/*
 * yolo2_light_b200_glue.c -- the reference-side binding a yolo2_light maintainer would add (see INTEGRATION.md).
 *
 * Compiled TOGETHER WITH the reference's own sources (it includes the reference's src/additionally.h) and linked
 * against libyolo2_light_b200.so.  It adds functions with exactly the shape of the reference's predict slots:
 *
 *     float *network_predict_b200(network net, float *input);              (network_predict_cpu / network_predict_gpu_cudnn)
 *     float *network_predict_b200_quantized(network net, float *input);    (network_predict_quantized, the CPU build's INT8
 *                                                 rule: conv i >= 1 without LINEAR activation, yolov2_forward_network_quantized.c:1036)
 *     float *network_predict_b200_cudnn_quantized(network net, float *input);   (network_predict_gpu_cudnn_quantized,
 *                                                 additionally.h:958: the GPU build's INT8 rule on the layers' own l.quantized,
 *                                                 what src/main.c:199-206 runs for a GPU build with -quantized)
 *     void   forward_convolutional_layer_b200(layer l, network_state state);      (slot of forward_convolutional_layer_cpu,
 *     void   forward_convolutional_layer_b200_q(layer l, network_state state);     additionally.h:925 / ..._q, :927: by-value layer)
 *     float *network_predict_b200_batch(network net, float *images, int nimg, int ngpus, int quantized);   (additive: many
 *                                                 images over the GPUs of the box from this one C process)
 *     detection *get_network_boxes_nms_b200(network *net, int w, int h, float thresh, float nms, int relative, int *num,
 *                                           int letter);      (optional: decode + NMS on the device)
 *     void   network_b200_set_xnor_rule(int rule);    (YB_XNOR_CPU / YB_XNOR_GPU for the handles built after the call: with
 *                                                 YB_XNOR_GPU, network_predict_b200 computes what network_predict_gpu_cudnn
 *                                                 computes on an XNOR network, and network_predict_b200_cudnn_quantized
 *                                                 what network_predict_gpu_cudnn_quantized does.  Until it is called, a
 *                                                 handle keeps the library's initial rule: YB_XNOR_RULE in the
 *                                                 environment, else YB_XNOR_CPU)
 *
 * Call sites to switch: src/main.c:199-219, src/main.c:394-414, src/additionally.c:4639-4659.
 * Preconditions are the reference's own (main.c:160-171): parse_network_cfg, load_weights_upto_cpu,
 * yolov2_fuse_conv_batchnorm, calculate_binary_weights, [quantinization_and_get_multipliers].
 *
 * On the first call the prepared per-layer arrays of `net` are handed to the engine as yb_layer_desc[]
 * (snapshot after preparation, SURVEY 8b); afterwards each call is H2D + CUDA graph + D2H.  The activated
 * YOLO/REGION tensors are copied into the reference layers' host l.output, so get_network_boxes / do_nms_sort /
 * draw_detections_v3 keep working unchanged.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "additionally.h"
#include "yolo2_light_b200.h"

#define YB_GLUE_MAX_NETS 16
static struct { layer *key; int quantized, xnor_rule; yb_network *h; unsigned long stamp; } g_nets[YB_GLUE_MAX_NETS];
static unsigned long g_stamp;   /* which handle of a net ran last: the decode must read THAT engine's tensors */
static int g_xnor_rule = -1;   /* the XNOR rule of the handles built from now on; -1: the library's initial rule */

void network_b200_set_xnor_rule(int rule)
{
    if (rule != YB_XNOR_CPU && rule != YB_XNOR_GPU) { fprintf(stderr, "network_b200_set_xnor_rule: bad rule %d\n", rule); exit(1); }
    g_xnor_rule = rule;
}

static yb_network *glue_build(network net, int quantized)
{
    yb_layer_desc *d = (yb_layer_desc *)calloc(net.n, sizeof(yb_layer_desc));
    int i;
    for (i = 0; i < net.n; ++i) {
        layer *l = &net.layers[i];
        d[i].type = (int)l->type;               /* same numeric values as LAYER_TYPE */
        d[i].activation = (int)l->activation;   /* same numeric values as ACTIVATION */
        d[i].batch_normalize = l->batch_normalize;
        d[i].h = l->h; d[i].w = l->w; d[i].c = l->c; d[i].n = l->n;
        d[i].size = l->size; d[i].stride = l->stride; d[i].pad = l->pad;
        d[i].out_h = l->out_h; d[i].out_w = l->out_w; d[i].out_c = l->out_c;
        d[i].xnor = l->xnor; d[i].quantized = l->quantized; d[i].index = l->index;
        d[i].classes = l->classes; d[i].coords = l->coords; d[i].softmax = l->softmax; d[i].total = l->total;
        d[i].reverse = l->reverse; d[i].scale = l->scale;
        d[i].input_layers = l->input_layers; d[i].mask = l->mask;
        if (l->type == CONVOLUTIONAL) {
            d[i].weights = l->weights; d[i].biases = l->biases;
            d[i].scales = l->scales; d[i].rolling_mean = l->rolling_mean; d[i].rolling_variance = l->rolling_variance;
            if (quantized) {
                d[i].weights_int8 = l->weights_int8;
                d[i].weights_quant_multipler = l->weights_quant_multipler;
                d[i].input_quant_multipler = l->input_quant_multipler;
            }
            d[i].mean_arr = l->xnor ? l->mean_arr : NULL;
        } else if (l->type == YOLO || l->type == REGION) {
            d[i].anchors = l->biases;
        }
    }
    yb_network *h = yb_network_from_layers(d, net.n, net.batch, net.h, net.w, net.c, quantized);
    free(d);
    if (h && net.gpu_index >= 0) yb_network_set_device(h, net.gpu_index);
    if (h && g_xnor_rule >= 0) yb_network_set_xnor_rule(h, g_xnor_rule);
    return h;
}

static yb_network *glue_handle(network net, int quantized)
{
    int k;
    for (k = 0; k < YB_GLUE_MAX_NETS; ++k)
        if (g_nets[k].h && g_nets[k].key == net.layers && g_nets[k].quantized == quantized && g_nets[k].xnor_rule == g_xnor_rule) {
            g_nets[k].stamp = ++g_stamp;
            return g_nets[k].h;
        }
    for (k = 0; k < YB_GLUE_MAX_NETS; ++k)
        if (!g_nets[k].h) {
            g_nets[k].h = glue_build(net, quantized);
            g_nets[k].key = net.layers; g_nets[k].quantized = quantized; g_nets[k].xnor_rule = g_xnor_rule; g_nets[k].stamp = ++g_stamp;
            return g_nets[k].h;
        }
    fprintf(stderr, "yolo2_light_b200 glue: more than %d (network, rules) triples -- raise YB_GLUE_MAX_NETS\n", YB_GLUE_MAX_NETS);
    exit(1);   /* the reference's error convention: message + exit */
}

static float *glue_predict(network net, float *input, int quantized)
{
    int i;
    yb_network *h = glue_handle(net, quantized);
    if (quantized == YB_QUANT_GPU) yb_network_predict_cudnn_quantized(h, input);
    else if (quantized) yb_network_predict_quantized(h, input);
    else yb_network_predict(h, input);
    /* what get_network_boxes reads (additionally.c:4391-4398): host l.output of every YOLO / REGION layer */
    for (i = 0; i < net.n; ++i) {
        layer *l = &net.layers[i];
        if (l->type == YOLO || l->type == REGION || i == net.n - 1) {
            int count = 0;
            const float *src = yb_network_layer_output(h, i, &count);
            if (src && l->output) memcpy(l->output, src, sizeof(float) * (size_t)count);
        }
    }
    for (i = net.n - 1; i > 0; --i) if (net.layers[i].type != COST) break;   /* as network_predict_cpu returns */
    return net.layers[i].output;
}

static int glue_find(network *net)   /* table slot of the handle of `net` that predicted last, or -1 */
{
    int k, best = -1;
    for (k = 0; k < YB_GLUE_MAX_NETS; ++k)
        if (g_nets[k].h && g_nets[k].key == net->layers && (best < 0 || g_nets[k].stamp > g_nets[best].stamp)) best = k;
    return best;
}

/*
 * Slot of the pair  dets = get_network_boxes(net, w, h, thresh, hier, map, relative, &n, letter);  do_nms_sort(dets, n,
 * classes, nms);  (src/main.c:228-229, :423-427): decode + NMS run on the device, on the tensors the last
 * network_predict_b200*(net, ...) left in HBM, and only the candidate rows come back.  Returns a `detection`
 * array laid out like make_network_boxes' (src/additionally.c:4238: prob[classes] per entry), to be released with the
 * reference's free_detections.  batch item 0, like the reference.  nms = 0 skips the suppression.
 */
detection *get_network_boxes_nms_b200(network *net, int w, int h, float thresh, float nms, int relative, int *num, int letter)
{
    const int slot = glue_find(net);
    yb_network *hnd;
    layer l = net->layers[net->n - 1];
    const int classes = l.classes, stride = 5 + classes, cap = 8192;
    float *rows;
    int *counts, n, i, quantized;
    detection *dets;
    if (slot < 0) { fprintf(stderr, "get_network_boxes_nms_b200: call network_predict_b200 first\n"); exit(1); }
    hnd = g_nets[slot].h; quantized = g_nets[slot].quantized;
    rows = (float *)malloc(sizeof(float) * (size_t)net->batch * cap * stride);
    counts = (int *)calloc(net->batch, sizeof(int));
    if (yb_network_detect(hnd, quantized, w, h, thresh, nms, relative, letter, rows, cap, counts) != stride) {
        fprintf(stderr, "get_network_boxes_nms_b200: %s\n", yb_last_error()); exit(1);
    }
    n = counts[0] < cap ? counts[0] : cap;
    dets = (detection *)calloc(n > 0 ? n : 1, sizeof(detection));
    for (i = 0; i < n; ++i) {
        const float *r = rows + (size_t)i * stride;
        dets[i].bbox.x = r[0]; dets[i].bbox.y = r[1]; dets[i].bbox.w = r[2]; dets[i].bbox.h = r[3];
        dets[i].objectness = r[4];
        dets[i].classes = classes;
        dets[i].prob = (float *)calloc(classes, sizeof(float));
        memcpy(dets[i].prob, r + 5, sizeof(float) * classes);
    }
    if (num) *num = n;
    free(rows); free(counts);
    return dets;
}

/*
 * Slot of forward_convolutional_layer_cpu(layer l, network_state state) (src/additionally.h:925, yolov2_forward_network.c:30)
 * and of forward_convolutional_layer_q (src/yolov2_forward_network_quantized.c:527): same by-value signature, reads
 * state.input (host, l.batch * l.c*l.h*l.w floats), writes the layer's host l.output.  The FP32 / XNOR choice follows l.xnor
 * like the reference; the _q form is the INT8 variant.  One single-layer engine per (layer, variant) is kept, keyed by the
 * layer's weight pointer.
 */
#define YB_GLUE_MAX_LAYERS 512
static struct { float *key; int variant; yb_network *h; } g_layers[YB_GLUE_MAX_LAYERS];

static void glue_forward_conv(layer l, network_state state, int variant)
{
    int k;
    yb_network *h = NULL;
    if (l.type != CONVOLUTIONAL) { fprintf(stderr, "forward_convolutional_layer_b200: not a convolutional layer\n"); exit(1); }
    for (k = 0; k < YB_GLUE_MAX_LAYERS && g_layers[k].h; ++k)
        if (g_layers[k].key == l.weights && g_layers[k].variant == variant) { h = g_layers[k].h; break; }
    if (!h) {
        network one;
        if (k == YB_GLUE_MAX_LAYERS) { fprintf(stderr, "forward_convolutional_layer_b200: layer table full\n"); exit(1); }
        memset(&one, 0, sizeof(one));
        one.n = 1; one.layers = &l; one.batch = l.batch; one.h = l.h; one.w = l.w; one.c = l.c; one.gpu_index = state.net.layers ? state.net.gpu_index : -1;
        h = glue_build(one, variant);
        if (variant) yb_network_set_option(h, "q_index_offset", 1);   /* the `i >= 1` half of the INT8 rule lives in the caller's loop */
        g_layers[k].key = l.weights; g_layers[k].variant = variant; g_layers[k].h = h;
    }
    yb_forward_convolutional_layer(h, 0, variant, state.input, l.output);
}
void forward_convolutional_layer_b200(layer l, network_state state) { glue_forward_conv(l, state, 0); }
void forward_convolutional_layer_b200_q(layer l, network_state state) { glue_forward_conv(l, state, 1); }

/*
 * Batch extension (SURVEY 8b): `nimg` images (host NCHW float) over `ngpus` GPUs from this one process; weights are built on
 * the first device and broadcast once.  Afterwards *per-image* results are read with yb_network_batch_output through the
 * handle returned by network_b200_handle (the reference's layers hold room for net.batch images only).  Returns the last
 * layer's results, nimg x outputs floats.
 */
yb_network *network_b200_handle(network net, int quantized) { return glue_handle(net, quantized); }
float *network_predict_b200_batch(network net, float *images, int nimg, int ngpus, int quantized)
{
    yb_network *h = glue_handle(net, quantized);
    if (yb_network_predict_batch(h, images, nimg, ngpus, quantized) != 0) { fprintf(stderr, "network_predict_b200_batch: %s\n", yb_last_error()); exit(1); }
    return (float *)yb_network_batch_output(h, net.n - 1, NULL);
}

float *network_predict_b200(network net, float *input) { return glue_predict(net, input, 0); }
float *network_predict_b200_quantized(network net, float *input) { return glue_predict(net, input, YB_QUANT_CPU); }
float *network_predict_b200_cudnn_quantized(network net, float *input) { return glue_predict(net, input, YB_QUANT_GPU); }
