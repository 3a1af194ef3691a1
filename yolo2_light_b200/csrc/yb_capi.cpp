// yb_capi.cpp -- the extern "C" surface declared in include/yolo2_light_b200.h
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "yb_engine.h"
#include "yb_model.h"

using namespace yb;

static thread_local std::string g_last_error;
static int g_abort_on_error = 1;

static void report(const std::string &msg) {
    g_last_error = msg;
    if (g_abort_on_error) {   // reference convention: print and die (additionally.c:1595-1600)
        fprintf(stderr, "yolo2_light_b200: %s\n", msg.c_str());
        abort();
    }
}

#define YB_TRY try {
#define YB_CATCH(retval)                                                       \
    }                                                                          \
    catch (const yb::Error &e) { report(e.msg); return retval; }               \
    catch (const std::exception &e) { report(e.what()); return retval; }
#define YB_CATCH_VOID                                                          \
    }                                                                          \
    catch (const yb::Error &e) { report(e.msg); return; }                      \
    catch (const std::exception &e) { report(e.what()); return; }

// The options of an engine of `net` on `device`; upload == false leaves its weight arena to a broadcast.
static EngineOptions engine_options(const Network &net, int quantized, int device, bool upload) {
    EngineOptions opt;
    opt.device = device;
    opt.precision = net.precision;
    opt.rule = quant_rule(quantized);
    opt.xnor_rule = net.xnor_rule;
    opt.upload = upload;
    opt.fuse = net.fuse;
    opt.keep_counts = net.keep_counts;
    opt.q_index_offset = net.q_index_offset;
    return opt;
}

static Engine *get_engine(yb_network *n, int quantized, bool upload = true) {
    Network &net = n->net;
    const int slot = quant_rule(quantized);
    if (!net.engine[slot]) net.engine[slot] = build_engine(&net, engine_options(net, quantized, net.device, upload));
    return net.engine[slot].get();
}

extern "C" {

void yb_set_abort_on_error(int on) { g_abort_on_error = on; }
const char *yb_last_error(void) { return g_last_error.c_str(); }
const char *yb_version(void) { return "yolo2_light_b200 0.1 (sm_90a)"; }

// The XNOR rule a new network starts with: YB_XNOR_RULE (0 or 1) when set, else YB_XNOR_CPU.  It lets a host program that
// builds its networks through unchanged code, such as the drop-in glue, choose the GPU build's XNOR arithmetic.
static int initial_xnor_rule() {
    const char *v = getenv("YB_XNOR_RULE");
    if (!v) return YB_XNOR_CPU;
    if (!strcmp(v, "0")) return YB_XNOR_CPU;
    if (!strcmp(v, "1")) return YB_XNOR_GPU;
    fatal_throw(std::string("YB_XNOR_RULE=") + v + ": must be 0 (YB_XNOR_CPU) or 1 (YB_XNOR_GPU)");
}

yb_network *yb_parse_network_cfg(const char *filename, int batch, int quantized) {
    YB_TRY
    const int xnor_rule = initial_xnor_rule();
    Network *net = parse_network_cfg(filename, batch, quantized);
    yb_network *h = new yb_network();
    h->net = std::move(*net);
    h->net.xnor_rule = xnor_rule;
    delete net;
    return h;
    YB_CATCH(nullptr)
}

int yb_load_weights_upto(yb_network *net, const char *filename, int cutoff) {
    YB_TRY
    load_weights_upto(&net->net, filename, cutoff);
    return 0;
    YB_CATCH(-1)
}

void yb_fuse_conv_batchnorm(yb_network *net) { YB_TRY fuse_conv_batchnorm(&net->net); YB_CATCH_VOID }
void yb_calculate_binary_weights(yb_network *net) { YB_TRY calculate_binary_weights(&net->net); YB_CATCH_VOID }
void yb_quantinization_and_get_multipliers(yb_network *net) {
    YB_TRY quantinization_and_get_multipliers(&net->net); YB_CATCH_VOID
}

yb_network *yb_network_from_layers(const yb_layer_desc *layers, int n_layers, int batch, int h, int w, int c,
                                   int quantized) {
    YB_TRY
    if (!layers || n_layers <= 0 || batch <= 0 || h <= 0 || w <= 0 || c <= 0) fatal_throw("from_layers: bad arguments");
    std::unique_ptr<yb_network> hold(new yb_network());   // released to the caller only when every layer validated
    yb_network *hnd = hold.get();
    Network &net = hnd->net;
    net.batch = batch; net.h = h; net.w = w; net.c = c; net.inputs = h * w * c; net.quantized = quantized;
    net.xnor_rule = initial_xnor_rule();
    net.layers.resize(n_layers);
    for (int i = 0; i < n_layers; ++i) {
        const yb_layer_desc &d = layers[i];
        Layer &l = net.layers[i];
        l.type = d.type; l.activation = d.activation; l.batch_normalize = d.batch_normalize;
        l.h = d.h; l.w = d.w; l.c = d.c; l.n = d.n; l.size = d.size; l.stride = d.stride; l.pad = d.pad;
        l.out_h = d.out_h; l.out_w = d.out_w; l.out_c = d.out_c;
        l.xnor = d.xnor; l.quantized = d.quantized; l.index = d.index;
        l.classes = d.classes; l.coords = d.coords; l.softmax = d.softmax; l.total = d.total;
        l.reverse = d.reverse; l.scale = d.scale;
        l.inputs = l.h * l.w * l.c;
        switch (l.type) {
        case YB_CONVOLUTIONAL: {
            const size_t nw = (size_t)l.n * l.c * l.size * l.size;
            if (!d.weights || !d.biases) fatal_throw("from_layers: conv without weights/biases");
            l.weights.assign(d.weights, d.weights + nw);
            l.biases.assign(d.biases, d.biases + l.n);
            if (l.batch_normalize) {
                if (!d.scales || !d.rolling_mean || !d.rolling_variance) fatal_throw("from_layers: BN arrays missing");
                l.scales.assign(d.scales, d.scales + l.n);
                l.rolling_mean.assign(d.rolling_mean, d.rolling_mean + l.n);
                l.rolling_variance.assign(d.rolling_variance, d.rolling_variance + l.n);
            }
            if (d.weights_int8) {
                l.weights_int8.assign(d.weights_int8, d.weights_int8 + nw);
                l.weights_quant_multipler = d.weights_quant_multipler;
                l.input_quant_multipler = d.input_quant_multipler;
                l.has_int8 = true;
            }
            if (d.mean_arr) { l.mean_arr.assign(d.mean_arr, d.mean_arr + l.n); l.has_mean_arr = true; }
            l.outputs = l.out_h * l.out_w * l.out_c;
            break;
        }
        case YB_ROUTE:
            if (!d.input_layers || l.n <= 0) fatal_throw("from_layers: route without input_layers");
            l.input_layers.assign(d.input_layers, d.input_layers + l.n);
            l.outputs = 0;
            for (int s : l.input_layers) {
                if (s < 0 || s >= i) fatal_throw("from_layers: bad route index");
                l.input_sizes.push_back(net.layers[s].outputs);
                l.outputs += net.layers[s].outputs;
            }
            break;
        case YB_YOLO:
            // the decoders index anchors[2 * mask[a]] for a < n: reject descriptions that would read out of bounds
            if (!d.mask || !d.anchors || l.n <= 0 || l.total <= 0) fatal_throw("from_layers: yolo layer without mask / anchors");
            l.mask.assign(d.mask, d.mask + l.n);
            for (int m : l.mask) if (m < 0 || m >= l.total) fatal_throw("from_layers: yolo mask entry out of range");
            l.anchors.assign(d.anchors, d.anchors + 2 * (size_t)l.total);
            if (i == 0 || l.c != l.n * (l.classes + 4 + 1) || net.layers[i - 1].out_c != l.c)
                fatal_throw("from_layers: yolo layer " + std::to_string(i) + " does not match its input's channel count");
            l.outputs = l.h * l.w * l.n * (l.classes + 4 + 1);
            break;
        case YB_REGION:
            if (!d.anchors || l.n <= 0) fatal_throw("from_layers: region layer without anchors");
            l.anchors.assign(d.anchors, d.anchors + 2 * (size_t)l.n);
            l.outputs = l.h * l.w * l.n * (l.classes + l.coords + 1);
            break;
        case YB_SHORTCUT:
            if (l.index < 0 || l.index >= i) fatal_throw("from_layers: bad shortcut index");
            l.outputs = l.out_h * l.out_w * l.out_c;
            break;
        default:
            l.outputs = l.out_h * l.out_w * l.out_c;
            break;
        }
    }
    return hold.release();
    YB_CATCH(nullptr)
}

void yb_free_network(yb_network *net) { delete net; }

int yb_network_num_layers(const yb_network *net) { return (int)net->net.layers.size(); }

void yb_network_dims(const yb_network *n, int *o) {
    const Network &net = n->net;
    o[0] = (int)net.layers.size(); o[1] = net.batch; o[2] = net.h; o[3] = net.w; o[4] = net.c; o[5] = net.inputs;
    o[6] = net.layers.empty() ? 0 : net.layers.back().outputs;
    o[7] = (int)net.input_calibration.size();
}

int yb_network_layer(const yb_network *n, int i, yb_layer_desc *d) {
    if (i < 0 || i >= (int)n->net.layers.size()) return -1;
    const Layer &l = n->net.layers[i];
    memset(d, 0, sizeof(*d));
    d->type = l.type; d->activation = l.activation; d->batch_normalize = l.batch_normalize;
    d->h = l.h; d->w = l.w; d->c = l.c; d->n = l.n; d->size = l.size; d->stride = l.stride; d->pad = l.pad;
    d->out_h = l.out_h; d->out_w = l.out_w; d->out_c = l.out_c;
    d->xnor = l.xnor; d->quantized = l.quantized; d->index = l.index;
    d->classes = l.classes; d->coords = l.coords; d->softmax = l.softmax; d->total = l.total;
    d->reverse = l.reverse; d->scale = l.scale;
    d->input_layers = l.input_layers.empty() ? nullptr : l.input_layers.data();
    d->mask = l.mask.empty() ? nullptr : l.mask.data();
    d->anchors = l.anchors.empty() ? nullptr : l.anchors.data();
    d->weights = l.weights.empty() ? nullptr : l.weights.data();
    d->biases = l.biases.empty() ? nullptr : l.biases.data();
    d->scales = l.scales.empty() ? nullptr : l.scales.data();
    d->rolling_mean = l.rolling_mean.empty() ? nullptr : l.rolling_mean.data();
    d->rolling_variance = l.rolling_variance.empty() ? nullptr : l.rolling_variance.data();
    d->weights_int8 = l.has_int8 ? l.weights_int8.data() : nullptr;
    d->weights_quant_multipler = l.weights_quant_multipler;
    d->input_quant_multipler = l.input_quant_multipler;
    d->mean_arr = l.has_mean_arr ? l.mean_arr.data() : nullptr;
    return 0;
}

int yb_network_layer_outputs(const yb_network *n, int i) {
    if (i < 0 || i >= (int)n->net.layers.size()) return -1;
    return n->net.layers[i].outputs;
}

const float *yb_network_input_calibration(const yb_network *n, int *count) {
    if (count) *count = (int)n->net.input_calibration.size();
    return n->net.input_calibration.empty() ? nullptr : n->net.input_calibration.data();
}

void yb_set_batch_network(yb_network *net, int batch) { set_batch(&net->net, batch); }

int yb_network_set_device(yb_network *n, int device) {
    n->net.device = device;
    drop_engines(&n->net);
    return 0;
}
int yb_network_set_precision(yb_network *n, int precision) {
    if (precision != YB_PREC_BF16_TC && precision != YB_PREC_FP32) { report("bad precision"); return -1; }
    n->net.precision = precision;
    drop_engines(&n->net);
    return 0;
}
int yb_network_set_xnor_rule(yb_network *n, int rule) {
    if (rule != YB_XNOR_CPU && rule != YB_XNOR_GPU) { report("bad XNOR rule"); return -1; }
    n->net.xnor_rule = rule;
    drop_engines(&n->net);
    return 0;
}
/* diagnostic switches (tests): fusion on/off, keep raw integer results, INT8 rule index offset */
int yb_network_set_option(yb_network *n, const char *name, int value) {
    Network &net = n->net;
    if (!strcmp(name, "fuse")) net.fuse = value != 0;
    else if (!strcmp(name, "keep_counts")) net.keep_counts = value != 0;
    else if (!strcmp(name, "q_index_offset")) net.q_index_offset = value;
    else { report(std::string("unknown option ") + name); return -1; }
    drop_engines(&net);
    return 0;
}

int yb_network_set_letterbox(yb_network *n, int on) {
    n->net.letterbox = on != 0;   // read by each frame call when it fills its geometry table: no engine rebuild
    return 0;
}

long yb_network_get_info(yb_network *n, int quantized, const char *key) {
    YB_TRY
    return engine_info(get_engine(n, quantized), key);
    YB_CATCH(-1)
}

int yb_network_tc_plan(yb_network *n, int quantized, int layer, int *fields, int count) {
    YB_TRY
    return engine_tc_plan(get_engine(n, quantized), layer, fields, count);
    YB_CATCH(-1)
}

static float *predict_common(yb_network *n, const float *input, int quantized) {
    Engine *e = get_engine(n, quantized);
    engine_upload_input(e, input, nullptr);
    engine_forward(e, nullptr, nullptr);
    engine_download_outputs(e, &n->net, nullptr);
    n->net.last_launches = engine_num_launches(e);
    return n->net.layers.back().output;
}

float *yb_network_predict(yb_network *n, const float *input) {
    YB_TRY return predict_common(n, input, 0); YB_CATCH(nullptr)
}
float *yb_network_predict_quantized(yb_network *n, const float *input) {
    YB_TRY return predict_common(n, input, YB_QUANT_CPU); YB_CATCH(nullptr)
}
float *yb_network_predict_cudnn_quantized(yb_network *n, const float *input) {
    YB_TRY return predict_common(n, input, YB_QUANT_GPU); YB_CATCH(nullptr)
}

int yb_network_submit(yb_network *n, const float *input, int quantized) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    const int t = engine_submit(e, input);
    n->net.last_launches = engine_num_launches(e);
    return t;
    YB_CATCH(-1)
}
int yb_network_collect(yb_network *n, int ticket, int quantized) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    engine_collect(e, &n->net, ticket);
    return 0;
    YB_CATCH(-1)
}

}  // extern "C"

// With letterboxing on, a frame whose letterbox size has a side below 2 is refused: resize_image divides by that side
// minus 1 (additionally.c:3027-3028).
static void check_letterbox(const Network &net, const std::string &fb, int w, int h) {
    if (!net.letterbox) return;
    int nw, nh;
    letterbox_size(net.w, net.h, w, h, &nw, &nh);
    if (nw < 2 || nh < 2)
        fatal_throw(fb + " (" + std::to_string(w) + "x" + std::to_string(h) + ") letterboxes to " + std::to_string(nw) + "x" +
                    std::to_string(nh) + " in the " + std::to_string(net.w) + "x" + std::to_string(net.h) +
                    " network; letterboxing needs at least 2 pixels on each side");
}

// Argument checks of the frame entry points, all before any device work.
static void check_nimg(const Network &net, const std::string &f, int nimg) {
    if (nimg < 1 || nimg > net.batch)
        fatal_throw(f + ": nimg " + std::to_string(nimg) + " outside 1.." + std::to_string(net.batch) + " (net.batch)");
}
// The decode-only call, which takes sizes alone.
static void check_sizes(const Network &net, const char *fn, const int *w, const int *h, int nimg) {
    const std::string f(fn);
    check_nimg(net, f, nimg);
    if (!w || !h) fatal_throw(f + ": null w / h array");
    for (int b = 0; b < nimg; ++b)
        if (w[b] < 1 || h[b] < 1)
            fatal_throw(f + ": frame " + std::to_string(b) + " has size " + std::to_string(w[b]) + "x" + std::to_string(h[b]));
}
static void check_max_rows(const char *fn, int max_rows) {
    if (max_rows <= 0 || max_rows > DET_MAX_ROWS)
        fatal_throw(std::string(fn) + ": max_rows must be in 1.." + std::to_string(DET_MAX_ROWS));
}
// The frame calls: everything but the memory kind of device frames (check_frame_memory), without touching the device.
static void check_frames(const Network &net, const char *fn, const FrameBatch &batch) {
    const std::string f(fn);
    check_nimg(net, f, batch.nimg);
    if (!batch.frames) fatal_throw(f + ": null frames array");
    const int format = batch.fmt;
    if (format < YB_FRAME_RGB || format > YB_FRAME_NV12) fatal_throw(f + ": unknown frame format " + std::to_string(format));
    if (!batch.host && net.c != 3)
        fatal_throw(f + ": device frames have 3 channels, the network's input has " + std::to_string(net.c));
    const bool nv12 = format == YB_FRAME_NV12;
    for (int b = 0; b < batch.nimg; ++b) {
        const yb_device_frame &d = batch.frames[b];
        const std::string fb = f + ": frame " + std::to_string(b);
        if (!d.data) fatal_throw(fb + " is null");
        if (nv12 && !d.chroma) fatal_throw(fb + " has a null chroma plane");
        if (d.w < 1 || d.h < 1) fatal_throw(fb + " has size " + std::to_string(d.w) + "x" + std::to_string(d.h));
        if (nv12 && (d.w % 2 || d.h % 2))
            fatal_throw(fb + " has size " + std::to_string(d.w) + "x" + std::to_string(d.h) + ", NV12 needs an even width and height");
        // net.c bytes per packed pixel: 3 for device frames
        const long long row = format == YB_FRAME_RGB || format == YB_FRAME_BGR ? (long long)net.c * d.w : d.w;
        const long long pitch = batch.host ? row : d.pitch;   // host frames are packed (host_frame)
        if (pitch < row)
            fatal_throw(fb + " has pitch " + std::to_string(pitch) + " below its row of " + std::to_string(row) + " bytes");
        long long span = (d.h - 1) * pitch + row;   // the resize indexes within a frame in 32 bits
        if (format == YB_FRAME_RGB_PLANAR) {
            if (d.plane_stride < pitch * d.h)
                fatal_throw(fb + " has plane_stride " + std::to_string(d.plane_stride) + " below pitch * h = " +
                            std::to_string(pitch * d.h));
            span += 2 * d.plane_stride;
        }
        if (span > INT_MAX) fatal_throw(fb + (batch.host ? " has" : " addresses") + " more than INT_MAX bytes");
        check_letterbox(net, fb, d.w, d.h);
    }
}

// A host frame of w x h pixels of net.c bytes as an RGB frame of pitch w * net.c.  A frame whose pitch is not an int is
// refused by check_frames (by its size or its span); its pitch is left 0.
static yb_device_frame host_frame(const Network &net, const unsigned char *data, int w, int h) {
    const long long pitch = (long long)w * net.c;
    return yb_device_frame{data, nullptr, w, h, pitch > 0 && pitch <= INT_MAX ? (int)pitch : 0, 0};
}

// The frames of a host frame call as a batch
struct HostFrames {
    std::vector<yb_device_frame> table;
    FrameBatch batch{};
    // nimg frames, frame b w[b] x h[b]; the arrays are read once nimg, w and h have passed, and a null frames array is left
    // to check_frames
    HostFrames(const Network &net, const char *fn, const unsigned char *const *frames, const int *w, const int *h, int nimg) {
        check_nimg(net, fn, nimg);
        if (!w || !h) fatal_throw(std::string(fn) + ": null w / h array");
        for (int b = 0; frames && b < nimg; ++b) table.push_back(host_frame(net, frames[b], w[b], h[b]));
        batch = FrameBatch{frames ? table.data() : nullptr, nimg, YB_FRAME_RGB, true};
    }
    // net.batch frames of one size, stacked
    HostFrames(const Network &net, const unsigned char *images_hwc, int w, int h) {
        for (int b = 0; b < net.batch; ++b) table.push_back(host_frame(net, images_hwc + (size_t)b * w * h * net.c, w, h));
        batch = FrameBatch{table.data(), net.batch, YB_FRAME_RGB, true};
    }
};

// The synchronous and the pipelined frame call: checks, then the resize and the forward (+ decode and NMS).
static float *predict_frames(yb_network *n, const char *fn, const FrameBatch &b, int quantized, void *stream) {
    Network &net = n->net;
    check_frames(net, fn, b);
    if (!b.host) check_frame_memory(net.device, fn, b);
    Engine *e = get_engine(n, quantized);
    engine_upload_frames(e, &net, b, stream);
    engine_forward(e, nullptr, nullptr);
    engine_download_outputs(e, &net, nullptr);
    net.last_launches = engine_num_launches(e) + 1;   // + resize
    return net.layers.back().output;
}
// The drawing call's own checks: frames drawn in place must be distinct, and the colour index of every class must fit an int.
static void check_draw(const Network &net, const char *fn, const FrameBatch &b) {
    const std::string f(fn);
    for (int i = 0; i < b.nimg; ++i)
        for (int j = 0; j < i; ++j)
            if (b.frames[i].data == b.frames[j].data)
                fatal_throw(f + ": frames " + std::to_string(j) + " and " + std::to_string(i) + " share their data pointer");
    for (const Layer &l : net.layers)
        if ((l.type == YB_YOLO || l.type == YB_REGION) && l.classes > 17395)
            fatal_throw(f + ": " + std::to_string(l.classes) + " classes, drawing takes at most 17395 (cls * 123457 must fit an int)");
}
static int submit_frames(yb_network *n, const char *fn, const FrameBatch &b, int quantized, float thresh, float nms,
                         int relative, int letter, int max_rows, void *stream, bool draw = false) {
    Network &net = n->net;
    check_frames(net, fn, b);
    check_max_rows(fn, max_rows);
    if (draw) check_draw(net, fn, b);
    if (!b.host) check_frame_memory(net.device, fn, b);
    Engine *e = get_engine(n, quantized);
    const int t = engine_submit_frames(e, &net, b, thresh, nms, relative, letter, max_rows, stream, draw);
    net.last_launches = engine_num_launches(e) + 5 + (draw ? 2 : 0);   // + resize, count, emit, iou, nms (+ select, draw)
    return t;
}

extern "C" {

int yb_network_submit_u8(yb_network *n, const unsigned char *images_hwc, int w, int h, int quantized, float thresh, float nms,
                         int relative, int letter, int max_rows) {
    YB_TRY
    if (w <= 0 || h <= 0 || !images_hwc) fatal_throw("submit_u8: bad image");
    const HostFrames u(n->net, images_hwc, w, h);
    return submit_frames(n, "submit_frames_u8", u.batch, quantized, thresh, nms, relative, letter, max_rows, nullptr);
    YB_CATCH(-1)
}
int yb_network_submit_frames_u8(yb_network *n, const unsigned char *const *frames, const int *w, const int *h, int nimg,
                                int quantized, float thresh, float nms, int relative, int letter, int max_rows) {
    YB_TRY
    const HostFrames hf(n->net, "submit_frames_u8", frames, w, h, nimg);
    return submit_frames(n, "submit_frames_u8", hf.batch, quantized, thresh, nms, relative, letter, max_rows, nullptr);
    YB_CATCH(-1)
}
int yb_network_collect_detections(yb_network *n, int ticket, int quantized, const float **rows, const int **counts,
                                  size_t *d2h_bytes) {
    YB_TRY
    return engine_collect_detections(get_engine(n, quantized), ticket, rows, counts, d2h_bytes);
    YB_CATCH(-1)
}

float *yb_network_predict_image_u8(yb_network *n, const unsigned char *images_hwc, int w, int h, int quantized) {
    YB_TRY
    if (w <= 0 || h <= 0) fatal_throw("predict_image_u8: bad image size");
    const HostFrames u(n->net, images_hwc, w, h);
    return predict_frames(n, "predict_frames_u8", u.batch, quantized, nullptr);
    YB_CATCH(nullptr)
}
float *yb_network_predict_frames_u8(yb_network *n, const unsigned char *const *frames, const int *w, const int *h, int nimg,
                                    int quantized) {
    YB_TRY
    const HostFrames hf(n->net, "predict_frames_u8", frames, w, h, nimg);
    return predict_frames(n, "predict_frames_u8", hf.batch, quantized, nullptr);
    YB_CATCH(nullptr)
}
float *yb_network_predict_device_frames(yb_network *n, const yb_device_frame *frames, int nimg, int format, int quantized,
                                        void *stream) {
    YB_TRY
    return predict_frames(n, "predict_device_frames", FrameBatch{frames, nimg, format, false}, quantized, stream);
    YB_CATCH(nullptr)
}
int yb_network_submit_device_frames(yb_network *n, const yb_device_frame *frames, int nimg, int format, int quantized,
                                    float thresh, float nms, int relative, int letter, int max_rows, void *stream) {
    YB_TRY
    return submit_frames(n, "submit_device_frames", FrameBatch{frames, nimg, format, false}, quantized, thresh, nms, relative,
                         letter, max_rows, stream);
    YB_CATCH(-1)
}
int yb_network_submit_device_frames_draw(yb_network *n, const yb_device_frame *frames, int nimg, int format, int quantized,
                                         float thresh, float nms, int letter, int max_rows, void *stream) {
    YB_TRY
    return submit_frames(n, "submit_device_frames_draw", FrameBatch{frames, nimg, format, false}, quantized, thresh, nms, 1,
                         letter, max_rows, stream, true);
    YB_CATCH(-1)
}
// The list of the drawing ticket most recently collected under this number, of whichever engine collected it.
int yb_network_selected_detections(yb_network *n, int ticket, const yb_detection **dets, const int **counts) {
    YB_TRY
    unsigned long long best = 0;
    for (const std::shared_ptr<Engine> &e : n->net.engine) {
        const yb_detection *d = nullptr; const int *c = nullptr; unsigned long long seq = 0;
        if (e && engine_selected_detections(e.get(), ticket, &d, &c, &seq) == 0 && seq > best) {
            best = seq;
            if (dets) *dets = d;
            if (counts) *counts = c;
        }
    }
    return best ? 0 : -1;
    YB_CATCH(-1)
}
/* diagnostic: the resized planar float images the device pipeline produced for the last predict_image_u8 */
int yb_network_fetch_input(yb_network *n, int quantized, float *dst) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    engine_fetch_input(e, dst);
    return 0;
    YB_CATCH(-1)
}

const float *yb_network_layer_output(const yb_network *n, int i, int *count) {
    if (i < 0 || i >= (int)n->net.layers.size()) return nullptr;
    if (count) *count = (int)n->net.layers[i].output_count;
    return n->net.layers[i].output;
}

int yb_network_forward_device(yb_network *n, const void *d_input, int quantized, void *stream) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    engine_forward(e, d_input, stream);
    n->net.last_launches = engine_num_launches(e);
    return 0;
    YB_CATCH(-1)
}
int yb_network_sync_outputs(yb_network *n, int quantized, void *stream) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    engine_download_outputs(e, &n->net, stream);
    return 0;
    YB_CATCH(-1)
}

int yb_network_fetch_layer(yb_network *n, int i, int quantized, float *dst) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    engine_fetch_layer(e, &n->net, i, dst);
    return 0;
    YB_CATCH(-1)
}
int yb_network_fetch_counts(yb_network *n, int i, int quantized, int32_t *dst, size_t count) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    return engine_fetch_counts(e, i, dst, count);
    YB_CATCH(-1)
}

int yb_forward_convolutional_layer(yb_network *n, int i, int variant, const float *input, float *output) {
    YB_TRY
    const Network &src = n->net;
    if (i < 0 || i >= (int)src.layers.size() || src.layers[i].type != YB_CONVOLUTIONAL)
        fatal_throw("yb_forward_convolutional_layer: not a convolutional layer");
    if (!input || !output) fatal_throw("yb_forward_convolutional_layer: null buffer");
    const int rule = quant_rule(variant);
    const int key = 3 * i + rule;
    auto it = n->single.find(key);
    if (it == n->single.end() || it->second->net.batch != src.batch || it->second->net.device != src.device ||
        it->second->net.precision != src.precision) {
        std::unique_ptr<yb_network> tmp(new yb_network());
        Network &t = tmp->net;
        const Layer &l = src.layers[i];
        t.batch = src.batch; t.h = l.h; t.w = l.w; t.c = l.c; t.inputs = l.h * l.w * l.c;
        t.device = src.device; t.precision = src.precision; t.fuse = false;
        t.q_index_offset = i + src.q_index_offset;   // the `i >= 1` half of the CPU INT8 rule
        t.layers.push_back(l);
        // forward_convolutional_layer_gpu_cudnn_quantized runs the layer in INT8 whatever its l.quantized
        if (rule == YB_QUANT_GPU) t.layers[0].quantized = 1;
        t.layers[0].output = nullptr; t.layers[0].output_count = 0;
        it = n->single.insert_or_assign(key, std::move(tmp)).first;
    }
    yb_network *one = it->second.get();
    Engine *e = get_engine(one, rule);
    engine_upload_input(e, input, nullptr);
    engine_forward(e, nullptr, nullptr);
    engine_fetch_layer(e, &one->net, 0, output);
    return 0;
    YB_CATCH(-1)
}

/* ---- multi-GPU batch extension (SURVEY 8b "Batch extension", 8e) ------------------------------------------------------- */
int yb_network_set_devices(yb_network *n, const int *devices, int ndev) {
    YB_TRY
    if (ndev < 0 || (ndev > 0 && !devices)) fatal_throw("set_devices: bad arguments");
    const int have = engine_device_count();
    for (int k = 0; k < ndev; ++k)
        if (devices[k] < 0 || devices[k] >= have) fatal_throw("set_devices: device " + std::to_string(devices[k]) + " does not exist");
    n->devices.assign(devices, devices + ndev);
    for (auto &r : n->replicas) r.clear();
    if (ndev > 0 && n->net.device != devices[0]) { n->net.device = devices[0]; drop_engines(&n->net); }
    return 0;
    YB_CATCH(-1)
}

static std::vector<Engine *> get_replicas(yb_network *n, int quantized, int ngpus) {
    const int slot = quant_rule(quantized);
    if (n->devices.empty() || (int)n->devices.size() < ngpus) {
        const int have = engine_device_count();
        if (ngpus > have) fatal_throw("predict_batch: " + std::to_string(ngpus) + " GPUs requested, " + std::to_string(have) + " visible");
        n->devices.resize(ngpus);
        for (int k = 0; k < ngpus; ++k) n->devices[k] = k;
        for (auto &r : n->replicas) r.clear();
    }
    if (n->net.device != n->devices[0]) { n->net.device = n->devices[0]; drop_engines(&n->net); for (auto &r : n->replicas) r.clear(); }
    const bool fresh0 = !n->net.engine[slot];
    Engine *e0 = get_engine(n, quantized);
    if (fresh0) n->replicas[slot].clear();           // replica 0 was rebuilt: the others hold stale plans
    std::vector<std::shared_ptr<Engine>> &reps = n->replicas[slot];
    bool built = false;
    while ((int)reps.size() < ngpus - 1) {
        const int device = n->devices[reps.size() + 1];
        reps.push_back(build_engine(&n->net, engine_options(n->net, quantized, device, false)));   // weights arrive by the broadcast
        built = true;
    }
    std::vector<Engine *> all{e0};
    for (int k = 0; k + 1 < ngpus; ++k) all.push_back(reps[k].get());
    if (built) n->replication = engine_broadcast_arena(all);   // ONE collective, at init only
    return all;
}

int yb_network_predict_batch(yb_network *n, const float *images, int nimg, int ngpus, int quantized) {
    YB_TRY
    Network &net = n->net;
    if (!images || nimg <= 0 || ngpus <= 0) fatal_throw("predict_batch: bad arguments");
    const std::vector<Engine *> reps = get_replicas(n, quantized, ngpus);
    const int B = net.batch;
    const size_t per_img = (size_t)net.c * net.h * net.w;
    n->batch_out.assign(net.layers.size(), {});
    for (size_t i = 0; i < net.layers.size(); ++i) {
        const Layer &l = net.layers[i];
        if (l.type == YB_YOLO || l.type == YB_REGION || i + 1 == net.layers.size()) n->batch_out[i].assign((size_t)nimg * l.outputs, 0.f);
    }
    n->batch_nimg = nimg;
    struct Pending { int ticket, first, count; };
    std::vector<std::vector<Pending>> q(ngpus);
    std::vector<std::vector<float>> padded;          // partial last shards, kept alive until collected
    std::vector<const float *> ptrs; std::vector<size_t> counts;
    auto collect_oldest = [&](int g) {
        const Pending p = q[g].front();
        q[g].erase(q[g].begin());
        engine_collect_ptrs(reps[g], p.ticket, ptrs, counts);
        for (size_t i = 0; i < ptrs.size(); ++i) {
            if (!ptrs[i] || n->batch_out[i].empty()) continue;
            const size_t outs = (size_t)net.layers[i].outputs;
            memcpy(n->batch_out[i].data() + (size_t)p.first * outs, ptrs[i], sizeof(float) * outs * p.count);
        }
    };
    int shard = 0;
    for (int first = 0; first < nimg; first += B, ++shard) {
        const int g = shard % ngpus, cnt = std::min(B, nimg - first);
        if (q[g].size() == 3) collect_oldest(g);
        const float *src = images + (size_t)first * per_img;
        if (cnt < B) {   // contiguous shards of whole images; the tail is padded with zero images whose results are dropped
            padded.emplace_back((size_t)B * per_img, 0.f);
            memcpy(padded.back().data(), src, sizeof(float) * per_img * cnt);
            src = padded.back().data();
        }
        q[g].push_back(Pending{engine_submit(reps[g], src), first, cnt});
    }
    for (int g = 0; g < ngpus; ++g) while (!q[g].empty()) collect_oldest(g);
    net.last_launches = engine_num_launches(reps[0]);
    return 0;
    YB_CATCH(-1)
}

const float *yb_network_batch_output(const yb_network *n, int i, int *per_image) {
    if (i < 0 || i >= (int)n->batch_out.size() || n->batch_out[i].empty()) return nullptr;
    if (per_image) *per_image = n->net.layers[i].outputs;
    return n->batch_out[i].data();
}
const char *yb_network_replication(const yb_network *n) { return n->replication.c_str(); }

int yb_network_weight_arena(yb_network *n, int quantized, int upload, void **d_ptr, size_t *bytes) {
    YB_TRY
    Engine *e = get_engine(n, quantized, upload != 0);
    engine_weight_arena(e, d_ptr, bytes);
    return 0;
    YB_CATCH(-1)
}

int yb_network_last_launches(const yb_network *n) { return n->net.last_launches; }

int yb_network_profile(yb_network *n, int quantized, const void *d_input, int *layer_idx, int *op_kind,
                       float *ms, int max) {
    YB_TRY
    Engine *e = get_engine(n, quantized);
    return engine_profile(e, d_input, layer_idx, op_kind, ms, max);
    YB_CATCH(-1)
}
const char *yb_op_kind_name(int k) { return op_kind_name(k); }

int yb_network_op_kernels(yb_network *n, int quantized, int *layer_idx, int *op_kind, const char **name, int max) {
    YB_TRY
    return engine_op_kernels(get_engine(n, quantized), layer_idx, op_kind, name, max);
    YB_CATCH(-1)
}

int yb_get_network_boxes(const yb_network *n, int b, int w, int h, float thresh, float nms, int relative,
                         int letter, float *out, int max_rows) {
    YB_TRY
    return get_boxes(&n->net, b, w, h, thresh, nms, relative, letter, out, max_rows);
    YB_CATCH(-1)
}

int yb_network_detect(yb_network *n, int quantized, int w, int h, float thresh, float nms, int relative, int letter,
                      float *rows, int max_rows, int *counts) {
    YB_TRY
    const std::vector<int> ws(n->net.batch, w), hs(n->net.batch, h);
    return yb_network_detect_frames(n, quantized, ws.data(), hs.data(), n->net.batch, thresh, nms, relative, letter, rows,
                                    max_rows, counts);
    YB_CATCH(-1)
}
int yb_network_detect_frames(yb_network *n, int quantized, const int *w, const int *h, int nimg, float thresh, float nms,
                             int relative, int letter, float *rows, int max_rows, int *counts) {
    YB_TRY
    check_sizes(n->net, "detect_frames", w, h, nimg);
    check_max_rows("detect_frames", max_rows);
    return engine_detect(get_engine(n, quantized), &n->net, w, h, nimg, thresh, nms, relative, letter, rows, max_rows, counts);
    YB_CATCH(-1)
}

/* INT8 input calibration: one forward (FP32 rule) + per-convolution |input| histograms on the GPU + the reference's
 * KL search on the host.  multipliers[b * nconv + k] for image b and the k-th CONVOLUTIONAL layer. */
int yb_network_calibrate(yb_network *n, const float *input, float *multipliers, int max_values) {
    YB_TRY
    Network &net = n->net;
    struct FuseGuard {   // every layer input must exist in memory: fusion off for the calibration engine, restored on any exit
        Network &net; bool old;
        explicit FuseGuard(Network &n_) : net(n_), old(n_.fuse) { if (old) { net.fuse = false; drop_engines(&net); } }
        ~FuseGuard() { if (old) { net.fuse = true; drop_engines(&net); } }
    } guard(net);
    Engine *e = get_engine(n, 0);
    engine_upload_input(e, input, nullptr);
    engine_forward(e, nullptr, nullptr);
    int nconv = 0;
    for (const Layer &l : net.layers) nconv += l.type == YB_CONVOLUTIONAL;
    if (max_values < nconv * net.batch) fatal_throw("calibrate: multipliers[] too small");
    std::vector<uint32_t> hist(4096);
    for (int b = 0; b < net.batch; ++b) {
        int k = 0;
        for (size_t i = 0; i < net.layers.size(); ++i) {
            if (net.layers[i].type != YB_CONVOLUTIONAL) continue;
            // network_calibrate_cpu, yolov2_forward_network.c:784: entropy_calibration(state.input, l.inputs, 1.0 / 16, 4096)
            engine_input_histogram(e, &net, (int)i, b, 1.0f / 16, 4096, hist.data());
            multipliers[(size_t)b * nconv + k++] = entropy_from_histogram(hist.data(), 1.0f / 16, 4096);
        }
    }
    return nconv;
    YB_CATCH(-1)
}
/* the host half alone (histogram + KL search of one array), == entropy_calibration(src, size, bin_width, max_bin) */
float yb_entropy_calibration(const float *src, size_t size, float bin_width, int max_bin) {
    YB_TRY
    if (max_bin < 129 || max_bin > 1 << 20) fatal_throw("entropy_calibration: bad max_bin");
    std::vector<uint32_t> hist(max_bin);
    abs_histogram_host(src, size, bin_width, max_bin, hist.data());
    return entropy_from_histogram(hist.data(), bin_width, max_bin);
    YB_CATCH(-1.f)
}
/* histogram of the input of layer i for image b after the last forward (GPU), for tests */
int yb_network_input_histogram(yb_network *n, int quantized, int layer, int img, float bin_width, int max_bin, uint32_t *hist) {
    YB_TRY
    engine_input_histogram(get_engine(n, quantized), &n->net, layer, img, bin_width, max_bin, hist);
    return 0;
    YB_CATCH(-1)
}

int yb_map_evaluate(const float *rows, const int *rows_per_image, int nimages, int classes, const float *truth, int ntruth,
                    float iou_thresh, float thresh_calc_avg_iou, double *ap_per_class, double *map_out, float *stats) {
    YB_TRY
    return map_evaluate(rows, rows_per_image, nimages, classes, truth, ntruth, iou_thresh, thresh_calc_avg_iou,
                        ap_per_class, map_out, stats);
    YB_CATCH(-1)
}

/* pinned host memory for the end-to-end path (input images) */
void *yb_alloc_pinned(size_t bytes);
void yb_free_pinned(void *p);

}  // extern "C"
