// yb_model.cpp -- host-side model preparation: .cfg parser, .weights loader, BN folding, XNOR weight
// statistics, INT8 quantisation, detection decode.  Behavioural mirror of the reference host code
// (src/additionally.c, src/yolov2_forward_network_quantized.c, src/box.c); written from its semantics,
// not from its text.  Compile WITHOUT fast-math / fp-contraction: several results are compared bit-for-bit
// with the reference's scalar build.
#include "yb_model.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <utility>

namespace yb {

void fatal_throw(const std::string &msg) { throw Error{msg}; }

// Every host `Layer::output` points into pinned memory owned by an Engine: whenever the engines go, those pointers go
// with them (a stale non-null pointer would make get_boxes / yb_network_layer_output read freed memory).
void drop_engines(Network *net) {
    for (auto &e : net->engine) e.reset();
    for (Layer &l : net->layers) { l.output = nullptr; l.output_count = 0; }
}

// ------------------------------------------------------------------------------------------------------
// .cfg reader.  Grammar of read_cfg / read_option (additionally.c:3423-3457, :3282-3300): every blank
// (space, tab, CR, LF) is removed from a line first; '[' starts a section; '#', ';' and empty lines are
// skipped; other lines are key=value split at the first '='.  Look-ups return the FIRST occurrence of a key
// (option_find, additionally.c:3343).
// ------------------------------------------------------------------------------------------------------
namespace {

struct Section {
    std::string type;
    std::vector<std::pair<std::string, std::string>> opts;
    const char *find(const char *key) const {
        for (auto &kv : opts)
            if (kv.first == key) return kv.second.c_str();
        return nullptr;
    }
    int geti(const char *key, int def) const { const char *v = find(key); return v ? atoi(v) : def; }
    float getf(const char *key, float def) const { const char *v = find(key); return v ? (float)atof(v) : def; }
    std::string gets(const char *key, const char *def) const { const char *v = find(key); return v ? v : def; }
};

std::vector<Section> read_cfg(const char *filename) {
    FILE *fp = fopen(filename, "r");
    if (!fp) fatal_throw(std::string("Couldn't open file: ") + filename);   // file_error, additionally.c:1610
    std::vector<Section> secs;
    std::string line;
    int ch;
    auto flush = [&]() {
        std::string s;
        for (char c : line)
            if (c != ' ' && c != '\t' && c != '\n' && c != '\r') s.push_back(c);
        line.clear();
        if (s.empty() || s[0] == '#' || s[0] == ';') return;
        if (s[0] == '[') {
            secs.push_back(Section{s, {}});
            return;
        }
        size_t eq = s.find('=');
        if (eq == std::string::npos || eq + 1 >= s.size() || secs.empty()) return;   // "could parse" warning case
        secs.back().opts.emplace_back(s.substr(0, eq), s.substr(eq + 1));
    };
    while ((ch = fgetc(fp)) != EOF) {
        if (ch == '\n') flush();
        else line.push_back((char)ch);
    }
    flush();
    fclose(fp);
    return secs;
}

// comma list walkers with the reference's atoi/atof + strchr(',')+1 stepping (e.g. additionally.c:3612-3617)
std::vector<float> float_list(const char *a, int limit = -1) {
    std::vector<float> out;
    if (!a) return out;
    int n = 1;
    for (const char *p = a; *p; ++p) if (*p == ',') ++n;
    for (int i = 0; i < n && (limit < 0 || i < limit); ++i) {
        out.push_back((float)atof(a));
        const char *nx = strchr(a, ',');
        if (!nx) break;
        a = nx + 1;
    }
    return out;
}
std::vector<int> int_list(const char *a) {
    std::vector<int> out;
    if (!a) return out;
    int n = 1;
    for (const char *p = a; *p; ++p) if (*p == ',') ++n;
    for (int i = 0; i < n; ++i) {
        out.push_back(atoi(a));
        const char *nx = strchr(a, ',');
        if (!nx) break;
        a = nx + 1;
    }
    return out;
}

int activation_from(const std::string &s) {   // get_activation, additionally.h:108-124
    static const char *names[] = {"logistic", "relu", "relie", "linear", "ramp", "tanh", "plse",
                                  "leaky", "elu", "loggy", "stair", "hardtan", "lhtan"};
    for (int i = 0; i < 13; ++i)
        if (s == names[i]) return i;
    fprintf(stderr, "Couldn't find activation function %s, going with ReLU\n", s.c_str());
    return YB_RELU;
}

int layer_type_from(const std::string &t) {   // string_to_layer_type, additionally.c:3820-3838
    if (t == "[yolo]") return YB_YOLO;
    if (t == "[region]") return YB_REGION;
    if (t == "[conv]" || t == "[convolutional]") return YB_CONVOLUTIONAL;
    if (t == "[max]" || t == "[maxpool]") return YB_MAXPOOL;
    if (t == "[reorg]") return YB_REORG;
    if (t == "[upsample]") return YB_UPSAMPLE;
    if (t == "[shortcut]") return YB_SHORTCUT;
    if (t == "[soft]" || t == "[softmax]") return YB_SOFTMAX;
    if (t == "[route]") return YB_ROUTE;
    return YB_BLANK;
}

}  // namespace

// parse_network_cfg, additionally.c:3955-4084 (layer rules: parse_convolutional :3534, parse_maxpool :3698,
// parse_route :3762, parse_shortcut :3744, parse_upsample :3734, parse_reorg :3716, parse_yolo :3642,
// parse_region :3573; size rules from the make_*_layer constructors :2336-2722).
Network *parse_network_cfg(const char *filename, int batch, int quantized) {
    std::vector<Section> secs = read_cfg(filename);
    if (secs.empty()) fatal_throw("Config file has no sections");
    std::unique_ptr<Network> net(new Network());
    net->quantized = quantized;
    const Section &ns = secs[0];
    {   // parse_net_options, additionally.c:3858-3897 (only the keys the forward path reads)
        int b = ns.geti("batch", 1);
        int subdivs = ns.geti("subdivisions", 1);
        int time_steps = ns.geti("time_steps", 1);
        if (subdivs) b /= subdivs;
        b *= time_steps;
        net->batch = b;
        net->input_calibration = float_list(ns.find("input_calibration"));
        net->h = ns.geti("height", 0);
        net->w = ns.geti("width", 0);
        net->c = ns.geti("channels", 0);
        net->inputs = ns.geti("inputs", net->h * net->w * net->c);
        if (!net->inputs && !(net->h && net->w && net->c)) fatal_throw("No input parameters supplied");
    }
    if (batch > 0) net->batch = batch;

    int ph = net->h, pw = net->w, pc = net->c, pinputs = net->inputs;
    int pquant = quantized;
    const int nl = (int)secs.size() - 1;
    net->layers.resize(nl);
    for (int idx = 0; idx < nl; ++idx) {
        const Section &s = secs[idx + 1];
        Layer &l = net->layers[idx];
        const int lt = layer_type_from(s.type);
        l.type = lt;
        l.h = ph; l.w = pw; l.c = pc;
        if (lt == YB_CONVOLUTIONAL) {
            // INT8 flag latch: a conv whose successor's successor is [yolo] switches quantisation off for the
            // rest of the net (additionally.c:3996-4003)
            if (idx + 3 <= nl && layer_type_from(secs[idx + 3].type) == YB_YOLO) pquant = 0;
            l.n = s.geti("filters", 1);
            l.size = s.geti("size", 1);
            l.stride = s.geti("stride", 1);
            int pad = s.geti("pad", 0);
            int padding = s.geti("padding", 0);
            if (pad) padding = l.size / 2;
            l.pad = padding;
            l.activation = activation_from(s.gets("activation", "logistic"));
            if (!(ph && pw && pc)) fatal_throw("Layer before convolutional layer must output image.");
            l.batch_normalize = s.geti("batch_normalize", 0);
            l.binary = s.geti("binary", 0);
            l.xnor = s.geti("xnor", 0);
            l.use_bin_output = s.geti("bin_output", 0);
            int q = pquant;
            if (idx == 0 || l.activation == YB_LINEAR || (idx > 1 && l.stride > 1) || l.size == 1) q = 0;
            l.quantized = q;
            if (l.stride <= 0) fatal_throw("convolutional: stride must be positive");
            l.out_h = (l.h + 2 * l.pad - l.size) / l.stride + 1;
            l.out_w = (l.w + 2 * l.pad - l.size) / l.stride + 1;
            l.out_c = l.n;
            l.outputs = l.out_h * l.out_w * l.out_c;
            l.inputs = l.w * l.h * l.c;
            const size_t nw = (size_t)l.c * l.n * l.size * l.size;
            l.weights.assign(nw, 0.f);       // the reference random-inits here (additionally.c:2751); a network
            l.biases.assign(l.n, 0.f);       // without a .weights file is unusable anyway (SURVEY F3)
            if (l.batch_normalize) {
                l.scales.assign(l.n, 1.f);
                l.rolling_mean.assign(l.n, 0.f);
                l.rolling_variance.assign(l.n, 0.f);
            }
        } else if (lt == YB_MAXPOOL) {
            l.stride = s.geti("stride", 1);
            l.size = s.geti("size", l.stride);
            l.pad = s.geti("padding", l.size - 1);
            if (!(ph && pw && pc)) fatal_throw("Layer before maxpool layer must output image.");
            if (l.stride <= 0) fatal_throw("maxpool: stride must be positive");
            l.out_w = (l.w + l.pad - l.size) / l.stride + 1;
            l.out_h = (l.h + l.pad - l.size) / l.stride + 1;
            l.out_c = l.c;
            l.outputs = l.out_h * l.out_w * l.out_c;
            l.inputs = l.h * l.w * l.c;
        } else if (lt == YB_ROUTE) {
            l.h = l.w = l.c = 0;   // make_route_layer (additionally.c:2451) leaves the input dims unset
            const char *ls = s.find("layers");
            if (!ls) fatal_throw("Route Layer must specify input layers");
            l.input_layers = int_list(ls);
            l.n = (int)l.input_layers.size();
            int outputs = 0;
            for (int &id : l.input_layers) {
                if (id < 0) id = idx + id;
                if (id < 0 || id >= idx) fatal_throw("route: bad layer index");
                l.input_sizes.push_back(net->layers[id].outputs);
                outputs += net->layers[id].outputs;
            }
            l.outputs = l.inputs = outputs;
            const Layer &first = net->layers[l.input_layers[0]];
            l.out_w = first.out_w; l.out_h = first.out_h; l.out_c = first.out_c;
            for (int i = 1; i < l.n; ++i) {
                const Layer &nx = net->layers[l.input_layers[i]];
                if (nx.out_w == first.out_w && nx.out_h == first.out_h) l.out_c += nx.out_c;
                else l.out_h = l.out_w = l.out_c = 0;
            }
        } else if (lt == YB_SHORTCUT) {
            const char *f = s.find("from");
            if (!f) fatal_throw("shortcut: missing from=");
            int index = atoi(f);
            if (index < 0) index = idx + index;
            if (index < 0 || index >= idx) fatal_throw("shortcut: bad from index");
            const Layer &from = net->layers[index];
            // make_shortcut_layer (additionally.c:2373): l.w/h/c describe the `from` tensor, out_* the input
            l.w = from.out_w; l.h = from.out_h; l.c = from.out_c;
            l.out_w = pw; l.out_h = ph; l.out_c = pc;
            l.outputs = l.inputs = pw * ph * pc;
            l.index = index;
            l.activation = activation_from(s.gets("activation", "linear"));
        } else if (lt == YB_UPSAMPLE) {
            int stride = s.geti("stride", 2);
            l.out_w = l.w * stride; l.out_h = l.h * stride; l.out_c = l.c;
            if (stride < 0) { stride = -stride; l.reverse = 1; l.out_w = l.w / stride; l.out_h = l.h / stride; }
            l.stride = stride;
            l.outputs = l.out_w * l.out_h * l.out_c;
            l.inputs = l.w * l.h * l.c;
            l.scale = s.getf("scale", 1);
        } else if (lt == YB_REORG) {
            l.stride = s.geti("stride", 1);
            l.reverse = s.geti("reverse", 0);
            if (!(ph && pw && pc)) fatal_throw("Layer before reorg layer must output image.");
            if (l.stride <= 0) fatal_throw("reorg: stride must be positive");
            if (l.reverse) { l.out_w = l.w * l.stride; l.out_h = l.h * l.stride; l.out_c = l.c / (l.stride * l.stride); }
            else { l.out_w = l.w / l.stride; l.out_h = l.h / l.stride; l.out_c = l.c * (l.stride * l.stride); }
            l.outputs = l.out_h * l.out_w * l.out_c;
            l.inputs = l.h * l.w * l.c;
        } else if (lt == YB_YOLO) {
            l.classes = s.geti("classes", 20);
            l.total = s.geti("num", 1);
            int num = l.total;
            const char *m = s.find("mask");
            if (m) { l.mask = int_list(m); num = (int)l.mask.size(); }
            else { l.mask.resize(num); for (int i = 0; i < num; ++i) l.mask[i] = i; }
            l.n = num;
            for (int mk : l.mask)   // the decoders read anchors[2 * mask[a]] (the reference would read out of bounds here)
                if (mk < 0 || mk >= l.total) fatal_throw("yolo: mask entry " + std::to_string(mk) + " outside num=" + std::to_string(l.total));
            l.max_boxes = s.geti("max", 90);
            l.c = l.n * (l.classes + 4 + 1);
            l.out_w = l.w; l.out_h = l.h; l.out_c = l.c;
            l.outputs = l.inputs = l.h * l.w * l.n * (l.classes + 4 + 1);
            if (l.outputs != pinputs)
                fatal_throw("Error: l.outputs == params.inputs: filters= in the [convolutional]-layer doesn't "
                            "correspond to classes= or mask= in [yolo]-layer");
            l.anchors.assign((size_t)l.total * 2, .5f);
            std::vector<float> a = float_list(s.find("anchors"), l.total * 2);
            std::copy(a.begin(), a.end(), l.anchors.begin());
        } else if (lt == YB_REGION) {
            l.coords = s.geti("coords", 4);
            l.classes = s.geti("classes", 20);
            l.n = s.geti("num", 1);
            l.c = 0;               // make_region_layer (additionally.c:2551) sets h, w only
            l.outputs = l.inputs = l.h * l.w * l.n * (l.classes + l.coords + 1);
            if (l.outputs != pinputs) fatal_throw("region: l.outputs != params.inputs");
            l.softmax = s.geti("softmax", 0);
            l.max_boxes = s.geti("max", 30);
            if (s.find("tree")) fatal_throw("region: softmax_tree (YOLO9000) is outside the supported hot path");
            l.anchors.assign((size_t)l.n * 2, .5f);
            std::vector<float> a = float_list(s.find("anchors"));
            if (a.size() > l.anchors.size()) l.anchors.resize(a.size());   // the reference writes past n*2 here
            std::copy(a.begin(), a.end(), l.anchors.begin());
            // out_h/out_w/out_c stay 0 as in make_region_layer (additionally.c:2551)
        } else if (lt == YB_SOFTMAX) {
            fatal_throw("[softmax] layers are outside the supported hot path");
        } else {
            fprintf(stderr, "Type not recognized: %s\n", s.type.c_str());
            l.type = YB_BLANK;
        }
        l.dontload = s.geti("dontload", 0);
        l.dontloadscales = s.geti("dontloadscales", 0);
        ph = l.out_h; pw = l.out_w; pc = l.out_c; pinputs = l.outputs;
    }
    return net.release();
}

void set_batch(Network *net, int batch) {
    net->batch = batch;
    drop_engines(net);
}

// load_weights_upto_cpu + load_convolutional_weights_cpu, additionally.c:3459-3529.  Like the reference, short
// reads are not an error (the remaining arrays keep their previous contents).
void load_weights_upto(Network *net, const char *filename, int cutoff) {
    FILE *fp = fopen(filename, "rb");
    if (!fp) fatal_throw(std::string("Couldn't open file: ") + filename);
    int32_t major = 0, minor = 0, revision = 0;
    size_t r = 0;
    r += fread(&major, sizeof(int32_t), 1, fp);
    r += fread(&minor, sizeof(int32_t), 1, fp);
    r += fread(&revision, sizeof(int32_t), 1, fp);
    if ((major * 10 + minor) >= 2) {
        r += fread(&net->seen, sizeof(uint64_t), 1, fp);
    } else {
        int32_t iseen = 0;
        r += fread(&iseen, sizeof(int32_t), 1, fp);
        net->seen = (uint64_t)iseen;
    }
    for (int i = 0; i < (int)net->layers.size() && i < cutoff; ++i) {
        Layer &l = net->layers[i];
        if (l.dontload || l.type != YB_CONVOLUTIONAL) continue;
        r += fread(l.biases.data(), sizeof(float), l.n, fp);
        if (l.batch_normalize && !l.dontloadscales) {
            r += fread(l.scales.data(), sizeof(float), l.n, fp);
            r += fread(l.rolling_mean.data(), sizeof(float), l.n, fp);
            r += fread(l.rolling_variance.data(), sizeof(float), l.n, fp);
        }
        r += fread(l.weights.data(), sizeof(float), l.weights.size(), fp);
    }
    (void)r;
    fclose(fp);
    drop_engines(net);
}

// yolov2_fuse_conv_batchnorm, additionally.c:67-109.  Expression order kept: b - (s*m)/(sqrt(v)+1e-6),
// (w*s)/(sqrt(v)+1e-6), all in float.
void fuse_conv_batchnorm(Network *net) {
    for (Layer &l : net->layers) {
        if (l.type != YB_CONVOLUTIONAL || !l.batch_normalize) continue;
        const size_t fs = (size_t)l.size * l.size * l.c;
        for (int f = 0; f < l.n; ++f) {
            const float denom = sqrtf(l.rolling_variance[f]) + .000001f;
            l.biases[f] = l.biases[f] - l.scales[f] * l.rolling_mean[f] / denom;
            float *w = l.weights.data() + (size_t)f * fs;
            const float sc = l.scales[f];
            for (size_t i = 0; i < fs; ++i) w[i] = w[i] * sc / denom;
        }
        l.batch_normalize = 0;
    }
    drop_engines(net);
}

// calculate_binary_weights -> binary_align_weights -> binarize_weights / get_mean_array
// (additionally.c:306, :196, :113, :188).  What the forward needs from it: mean_arr[f] = (sum_t |w[f][t]|)/K
// accumulated in float in tap order; the sign bits (w > 0) are packed on the device side in whatever layout
// the kernel wants (the reference's 256-bit aligned rows are a CPU/AVX2 artefact).
void calculate_binary_weights(Network *net) {
    for (Layer &l : net->layers) {
        if (l.type != YB_CONVOLUTIONAL || !l.xnor) continue;
        const int k = l.size * l.size * l.c;
        l.mean_arr.assign(l.n, 0.f);
        for (int f = 0; f < l.n; ++f) {
            float mean = 0;
            const float *w = l.weights.data() + (size_t)f * k;
            for (int i = 0; i < k; ++i) mean = (float)((double)mean + fabs((double)w[i]));
            mean = mean / k;
            l.mean_arr[f] = fabsf(mean);   // |+-mean| of the first binarised weight
        }
        l.has_mean_arr = true;
    }
    drop_engines(net);
}

namespace {
// get_distribution + get_multiplier, yolov2_forward_network_quantized.c:35-87: histogram of the positive
// values over 32 power-of-two ranges starting at 2^-16, best window of `bits_length` consecutive ranges.
float get_multiplier(const float *arr, size_t n, int bits_length) {
    const int number_of_ranges = 32;
    const float start_range = 1.F / 65536;
    int count[32] = {0};
    for (size_t i = 0; i < n; ++i) {
        const float w = arr[i];
        float cur = start_range;
        for (int j = 0; j < number_of_ranges; ++j) {
            if (fabs((double)cur) <= (double)w && (double)w < fabs((double)(cur * 2))) count[j]++;
            cur *= 2;
        }
    }
    int max_count_range = 0, index_max_count = 0;
    for (int j = 0; j < number_of_ranges; ++j) {
        int counter = 0;
        for (int i = j; i < (j + bits_length) && i < number_of_ranges; ++i) counter += count[i];
        if (max_count_range < counter) { max_count_range = counter; index_max_count = j; }
    }
    return 1 / (start_range * powf(2.f, (float)index_max_count));
}
inline int max_abs(int src, int max_val) {   // yolov2_forward_network_quantized.c:23
    if (abs(src) > abs(max_val)) src = (src > 0) ? max_val : -max_val;
    return src;
}
}  // namespace

// quantinization_and_get_multipliers, yolov2_forward_network_quantized.c:1402-1494.
// weights_quant_multipler = get_multiplier(w, 8)/4; weights_int8 = clamp127(trunc(w*mult));
// input_quant_multipler = input_calibration[conv ordinal] or 40 (ordinal counts ALL convs).
void quantinization_and_get_multipliers(Network *net) {
    int counter = 0;
    for (Layer &l : net->layers) {
        if (l.type != YB_CONVOLUTIONAL) continue;
        const size_t ws = l.weights.size();
        l.weights_quant_multipler = get_multiplier(l.weights.data(), ws, 8) / 4;
        l.weights_int8.resize(ws);
        for (size_t i = 0; i < ws; ++i) {
            const float w = l.weights[i] * l.weights_quant_multipler;
            l.weights_int8[i] = (int8_t)max_abs((int)w, 127);
        }
        l.input_quant_multipler = (counter < (int)net->input_calibration.size()) ? net->input_calibration[counter] : 40;
        ++counter;
        l.has_int8 = true;
    }
    drop_engines(net);
}

// ------------------------------------------------------------------------------------------------------
// Detection decode + NMS for one batch item: get_network_boxes (additionally.c:4403), get_yolo_detections
// (:4328), custom_get_region_detections (:4363) -> get_region_boxes_cpu (yolov2_forward_network.c:664),
// correct_yolo_boxes (:4281), do_nms_sort (box.c:296).
// ------------------------------------------------------------------------------------------------------
namespace {
struct Det { float x, y, w, h, objectness; std::vector<float> prob; int sort_class = 0; int order = 0; };

float overlap(float x1, float w1, float x2, float w2) {
    float l1 = x1 - w1 / 2, l2 = x2 - w2 / 2;
    float left = l1 > l2 ? l1 : l2;
    float r1 = x1 + w1 / 2, r2 = x2 + w2 / 2;
    float right = r1 < r2 ? r1 : r2;
    return right - left;
}
float box_iou(const Det &a, const Det &b) {   // box.c:46-70
    float w = overlap(a.x, a.w, b.x, b.w), h = overlap(a.y, a.h, b.y, b.h);
    float inter = (w < 0 || h < 0) ? 0 : w * h;
    float uni = a.w * a.h + b.w * b.h - inter;
    return inter / uni;
}
}  // namespace

int get_boxes(const Network *net, int b, int w, int h, float thresh, float nms, int relative, int letter,
              float *out, int max_rows) {
    std::vector<Det> dets;
    const int netw = net->w, neth = net->h;
    int classes = 0;
    if (b < 0 || b >= net->batch) fatal_throw("get_boxes: batch item " + std::to_string(b) + " out of range");
    for (const Layer &l : net->layers) {
        if (l.type == YB_YOLO) {
            classes = l.classes;
            if (!l.output) fatal_throw("get_boxes: run predict first");
            const float *p = l.output + (size_t)b * l.outputs;
            const int hw = l.w * l.h;
            auto entry = [&](int n, int loc, int e) { return n * hw * (4 + l.classes + 1) + e * hw + loc; };
            for (int i = 0; i < hw; ++i) {
                const int row = i / l.w, col = i % l.w;
                for (int n = 0; n < l.n; ++n) {
                    const float objectness = p[entry(n, i, 4)];
                    if (!(objectness > thresh)) continue;
                    Det d;
                    const int bi = entry(n, i, 0);
                    d.x = (col + p[bi + 0 * hw]) / l.w;
                    d.y = (row + p[bi + 1 * hw]) / l.h;
                    d.w = (float)(exp((double)p[bi + 2 * hw]) * l.anchors[2 * l.mask[n]] / netw);
                    d.h = (float)(exp((double)p[bi + 3 * hw]) * l.anchors[2 * l.mask[n] + 1] / neth);
                    d.objectness = objectness;
                    d.prob.resize(l.classes);
                    for (int j = 0; j < l.classes; ++j) {
                        float prob = objectness * p[entry(n, i, 5 + j)];
                        d.prob[j] = (prob > thresh) ? prob : 0;
                    }
                    dets.push_back(std::move(d));
                }
            }
        } else if (l.type == YB_REGION) {
            classes = l.classes;
            if (!l.output) fatal_throw("get_boxes: run predict first");
            const float *p = l.output + (size_t)b * l.outputs;
            for (int i = 0; i < l.w * l.h; ++i) {
                const int row = i / l.w, col = i % l.w;
                for (int n = 0; n < l.n; ++n) {
                    const int index = i * l.n + n;
                    const int p_index = index * (l.classes + 5) + 4;
                    const float scale = p[p_index];
                    const int box_index = index * (l.classes + 5);
                    Det d;
                    // get_region_box_cpu, yolov2_forward_network.c:653-661: logistic_activate computes in double and returns
                    // float (additionally.h:85); the add and the divide are float operations
                    const float lx = (float)(1. / (1. + exp(-(double)p[box_index + 0])));
                    const float ly = (float)(1. / (1. + exp(-(double)p[box_index + 1])));
                    d.x = (col + lx) / l.w;
                    d.y = (row + ly) / l.h;
                    d.w = expf(p[box_index + 2]) * l.anchors[2 * n] / l.w;
                    d.h = expf(p[box_index + 3]) * l.anchors[2 * n + 1] / l.h;
                    d.objectness = 1;
                    d.prob.resize(l.classes);
                    const int class_index = index * (l.classes + 5) + 5;
                    for (int j = 0; j < l.classes; ++j) {
                        float prob = scale * p[class_index + j];
                        d.prob[j] = (prob > thresh) ? prob : 0;
                    }
                    dets.push_back(std::move(d));
                }
            }
        }
    }
    // correct_yolo_boxes, additionally.c:4281-4315
    int new_w = netw, new_h = neth;
    if (letter) {
        if (((float)netw / w) < ((float)neth / h)) { new_w = netw; new_h = (h * netw) / w; }
        else { new_h = neth; new_w = (w * neth) / h; }
    }
    for (Det &d : dets) {
        d.x = (float)((d.x - (netw - new_w) / 2. / netw) / ((float)new_w / netw));
        d.y = (float)((d.y - (neth - new_h) / 2. / neth) / ((float)new_h / neth));
        d.w *= (float)netw / new_w;
        d.h *= (float)neth / new_h;
        if (!relative) { d.x *= w; d.w *= w; d.y *= h; d.h *= h; }
    }
    // do_nms_sort, box.c:296-328: drop objectness==0 to the tail, then per class sort by prob and suppress
    if (nms > 0) {
        int total = (int)dets.size();
        int k = total - 1;
        for (int i = 0; i <= k; ++i) {
            if (dets[i].objectness == 0) { std::swap(dets[i], dets[k]); --k; --i; }
        }
        total = k + 1;
        // Equal probabilities (they do occur: bf16 activations collide) are ordered by position in the candidate list, for every
        // class -- the same rule as the device path (k_det_nms, yb_detect.cuh).  The reference leaves it to qsort (box.c:311),
        // whose tie order is unspecified and differs between C libraries.
        for (int i = 0; i < total; ++i) dets[i].order = i;
        for (int c = 0; c < classes; ++c) {
            for (int i = 0; i < total; ++i) dets[i].sort_class = c;
            std::sort(dets.begin(), dets.begin() + total, [c](const Det &a, const Det &b2) {
                return a.prob[c] > b2.prob[c] || (a.prob[c] == b2.prob[c] && a.order < b2.order);
            });
            for (int i = 0; i < total; ++i) {
                if (dets[i].prob[c] == 0) continue;
                for (int j = i + 1; j < total; ++j)
                    if (box_iou(dets[i], dets[j]) > nms) dets[j].prob[c] = 0;
            }
        }
    }
    const int stride = 5 + classes;
    int nout = std::min<int>((int)dets.size(), max_rows);
    for (int i = 0; i < nout; ++i) {
        float *o = out + (size_t)i * stride;
        o[0] = dets[i].x; o[1] = dets[i].y; o[2] = dets[i].w; o[3] = dets[i].h; o[4] = dets[i].objectness;
        for (int c = 0; c < classes; ++c) o[5 + c] = dets[i].prob[c];
    }
    return (int)dets.size();
}

// ------------------------------------------------------------------------------------------------------
// INT8 input calibration (SURVEY 8f row 3).  entropy_calibration, yolov2_forward_network_quantized.c:1292-1398, from
// the |x| histogram (hist[b] = #elements with lround(fabs(x) / bin_width) == b, saturated into the last bin -- the part
// that touches the data and runs on the GPU).  Types and conversions follow the C source (float histogram and P/Q
// arrays, uint64 "outliers" updated through float arithmetic, double log, float accumulator), so the multiplier is
// bit-identical to the reference's for the same histogram.
// ------------------------------------------------------------------------------------------------------
float entropy_from_histogram(const uint32_t *hist, float bin_width, int max_bin) {
    std::vector<float> m_array(max_bin, 0.f), H(max_bin), P(max_bin, 0.f), Q(max_bin, 0.f);
    float quant_Q[128];
    uint64_t quant_cnt[128];
    for (int j = 0; j < max_bin; ++j) {
        // the reference counts with `float++`: exact up to 2^24, stuck there afterwards
        H[j] = (float)std::min<uint32_t>(hist[j], 16777216u);
    }
    for (int i = 128; i < max_bin; ++i) {
        uint64_t outliers = 0;
        const int last_bin = i - 1;
        for (int j = 0; j <= last_bin; ++j) P[j] = 0;
        for (int j = 0; j < max_bin; ++j) {
            if (j <= last_bin) P[j] = H[j];
            else outliers = (uint64_t)((float)outliers + H[j]);      // `outliers += H_histogram[j]` (float arithmetic)
        }
        const float quant_expand_width = i / 128.0F;
        for (int j = 0; j < 128; ++j) { quant_Q[j] = 0; quant_cnt[j] = 0; }
        for (int j = 0; j < i; ++j) {
            int quant_bin = (int)lround((double)(j / quant_expand_width));
            if (quant_bin > 127) quant_bin = 127;
            quant_Q[quant_bin] += P[j];
            if (P[j] != 0) quant_cnt[quant_bin]++;
        }
        for (int j = 0; j < i; ++j) Q[j] = 0;
        for (int j = 0; j < i; ++j) {
            int quant_bin = (int)lround((double)(j / quant_expand_width));
            if (quant_bin > 127) quant_bin = 127;
            if (P[j] != 0) Q[j] = quant_Q[quant_bin] / (float)quant_cnt[quant_bin];
        }
        P[last_bin] = P[last_bin] + (float)outliers;                  // saturation
        float sum_P = 0, sum_Q = 0;
        for (int j = 0; j < i; ++j) { sum_P += P[j]; sum_Q += Q[j]; }
        for (int j = 0; j < i; ++j) { P[j] /= sum_P; Q[j] /= sum_Q; }
        for (int j = 0; j < i; ++j) {
            const float ratio = (P[j] + FLT_MIN) / (Q[j] + FLT_MIN);
            m_array[i] = (float)((double)m_array[i] + (double)P[j] * log((double)ratio));
        }
    }
    float m_index = 128, min_m = FLT_MAX;
    for (int i = 128; i < max_bin; ++i)
        if (m_array[i] < min_m) { min_m = m_array[i]; m_index = (float)i; }
    const float threshold = (float)(((double)m_index + 0.5) * (double)bin_width);
    return 127 / threshold;
}

// host histogram with the reference's binning (yolov2_forward_network_quantized.c:1308-1316); the GPU kernel
// k_abs_hist computes the same integers
void abs_histogram_host(const float *src, size_t n, float bin_width, int max_bin, uint32_t *hist) {
    const int last_bin = max_bin - 1;
    for (int j = 0; j < max_bin; ++j) hist[j] = 0;
    for (size_t j = 0; j < n; ++j) {
        const long bin_num = lround(fabs((double)src[j]) / (double)bin_width);
        hist[bin_num >= last_bin ? last_bin : (int)bin_num]++;
    }
}

// ------------------------------------------------------------------------------------------------------
// mAP accounting (SURVEY 8f row 4): the bookkeeping of validate_detector_map, additionally.c:4541-4898, on detection
// rows produced elsewhere (yb_network_detect / yb_get_network_boxes with w = h = 1, thresh .005, nms .45 as the
// reference uses, :4576-4577, :4657-4659).  Same matching rule (best IoU above iou_thresh with equal class, :4711-4722),
// same global ranking by confidence (:4784), same 11-point interpolated AP (:4848-4866), same precision / recall / F1 /
// average-IoU figures at thresh_calc_avg_iou (:4745-4760, :4872-4880).  The "difficult" list (:4724-4735) is not modelled.
// ------------------------------------------------------------------------------------------------------
namespace {
struct BoxProb { float x, y, w, h, p; int class_id, image_index, truth_flag, unique_truth_index; };
float iou_xywh(float ax, float ay, float aw, float ah, float bx, float by, float bw, float bh) {
    Det a, b;
    a.x = ax; a.y = ay; a.w = aw; a.h = ah; b.x = bx; b.y = by; b.w = bw; b.h = bh;
    return box_iou(a, b);
}
}  // namespace

int map_evaluate(const float *rows, const int *rows_per_image, int nimages, int classes, const float *truth /* [n][6]:
                 image, class, x, y, w, h */, int ntruth, float iou_thresh, float thresh_calc_avg_iou,
                 double *ap_per_class, double *map_out, float *stats /* precision, recall, f1, avg_iou, tp, fp, fn, ndet */) {
    const int stride = 5 + classes;
    std::vector<BoxProb> det;
    std::vector<int> truth_classes_count(classes, 0);
    int unique_truth_count = 0, tp_for_thresh = 0, fp_for_thresh = 0;
    float avg_iou = 0;
    // truths grouped per image, in file order
    std::vector<std::vector<const float *>> per_image(nimages);
    for (int j = 0; j < ntruth; ++j) {
        const int im = (int)truth[(size_t)j * 6];
        if (im < 0 || im >= nimages) fatal_throw("map_evaluate: truth image index out of range");
        const int id = (int)truth[(size_t)j * 6 + 1];
        if (id < 0 || id >= classes) fatal_throw("map_evaluate: truth class out of range");
        per_image[im].push_back(truth + (size_t)j * 6);
    }
    const float *r = rows;
    for (int image_index = 0; image_index < nimages; ++image_index) {
        const auto &tr = per_image[image_index];
        const int num_labels = (int)tr.size();
        for (const float *t : tr) truth_classes_count[(int)t[1]]++;
        const size_t checkpoint = det.size();
        for (int i = 0; i < rows_per_image[image_index]; ++i, r += stride) {
            for (int class_id = 0; class_id < classes; ++class_id) {
                const float prob = r[5 + class_id];
                if (!(prob > 0)) continue;
                BoxProb d{r[0], r[1], r[2], r[3], prob, class_id, image_index, 0, -1};
                int truth_index = -1;
                float max_iou = 0;
                for (int j = 0; j < num_labels; ++j) {
                    const float *t = tr[j];
                    const float cur = iou_xywh(r[0], r[1], r[2], r[3], t[2], t[3], t[4], t[5]);
                    if (cur > iou_thresh && class_id == (int)t[1] && cur > max_iou) { max_iou = cur; truth_index = unique_truth_count + j; }
                }
                if (truth_index > -1) { d.truth_flag = 1; d.unique_truth_index = truth_index; }
                det.push_back(d);
                if (prob > thresh_calc_avg_iou) {
                    bool found = false;
                    for (size_t z = checkpoint; z + 1 < det.size(); ++z)
                        if (det[z].unique_truth_index == truth_index) { found = true; break; }
                    if (truth_index > -1 && !found) { avg_iou += max_iou; ++tp_for_thresh; }
                    else ++fp_for_thresh;
                }
            }
        }
        unique_truth_count += num_labels;
    }
    if (tp_for_thresh + fp_for_thresh > 0) avg_iou = avg_iou / (tp_for_thresh + fp_for_thresh);
    // SORT(detections): descending confidence (qsort's tie order is unspecified; ties keep insertion order here)
    std::stable_sort(det.begin(), det.end(), [](const BoxProb &a, const BoxProb &b) { return (a.p - b.p) > 0; });
    const int n = (int)det.size();
    struct PR { double precision, recall; int tp, fp; };
    std::vector<std::vector<PR>> pr(classes, std::vector<PR>(std::max(n, 1), PR{0, 0, 0, 0}));
    std::vector<char> truth_flags(std::max(unique_truth_count, 1), 0);
    for (int rank = 0; rank < n; ++rank) {
        if (rank > 0)
            for (int c = 0; c < classes; ++c) { pr[c][rank].tp = pr[c][rank - 1].tp; pr[c][rank].fp = pr[c][rank - 1].fp; }
        const BoxProb &d = det[rank];
        if (d.truth_flag == 1) {
            if (!truth_flags[d.unique_truth_index]) { truth_flags[d.unique_truth_index] = 1; pr[d.class_id][rank].tp++; }
        } else {
            pr[d.class_id][rank].fp++;
        }
        for (int c = 0; c < classes; ++c) {
            const int tp = pr[c][rank].tp, fp = pr[c][rank].fp, fn = truth_classes_count[c] - tp;
            pr[c][rank].precision = (tp + fp) > 0 ? (double)tp / (double)(tp + fp) : 0;
            pr[c][rank].recall = (tp + fn) > 0 ? (double)tp / (double)(tp + fn) : 0;
        }
    }
    double mean_ap = 0;
    for (int c = 0; c < classes; ++c) {
        double avg_precision = 0;
        for (int point = 0; point < 11; ++point) {
            const double cur_recall = point * 0.1;
            double cur_precision = 0;
            for (int rank = 0; rank < n; ++rank)
                if (pr[c][rank].recall >= cur_recall && pr[c][rank].precision > cur_precision) cur_precision = pr[c][rank].precision;
            avg_precision += cur_precision;
        }
        avg_precision = avg_precision / 11;
        if (ap_per_class) ap_per_class[c] = avg_precision;
        mean_ap += avg_precision;
    }
    mean_ap = mean_ap / classes;
    if (map_out) *map_out = mean_ap;
    if (stats) {
        const float cur_precision = (float)tp_for_thresh / ((float)tp_for_thresh + (float)fp_for_thresh);
        const float cur_recall = (float)tp_for_thresh / ((float)tp_for_thresh + (float)(unique_truth_count - tp_for_thresh));
        stats[0] = cur_precision; stats[1] = cur_recall;
        stats[2] = 2.F * cur_precision * cur_recall / (cur_precision + cur_recall);
        stats[3] = avg_iou; stats[4] = (float)tp_for_thresh; stats[5] = (float)fp_for_thresh;
        stats[6] = (float)(unique_truth_count - tp_for_thresh); stats[7] = (float)n;
    }
    return n;
}

}  // namespace yb
