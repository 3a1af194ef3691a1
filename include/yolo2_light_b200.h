/*
 * yolo2_light_b200.h -- C ABI of libyolo2_light_b200.so
 *
 * A Hopper (sm_90a, H100) forward-inference engine for darknet YOLO v2/v3 networks that sits behind the C surface
 * of AlexeyAB/yolo2_light.  Every entry point below names the reference interface it replaces (file:line relative
 * to the reference tree).  Plain pointers and sizes only; no CUDA, torch or C++ types cross this boundary.
 *
 * Two ways in:
 *   (1) stand-alone: yb_parse_network_cfg -> yb_load_weights_upto -> yb_fuse_conv_batchnorm ->
 *       yb_calculate_binary_weights -> [yb_quantinization_and_get_multipliers] -> yb_network_predict*
 *       (the exact call sequence of the reference app, src/main.c:160-219);
 *   (2) drop-in behind the reference's own parser/loader: the host program keeps its `network` and hands the
 *       prepared per-layer arrays over as yb_layer_desc[] (yb_network_from_layers); see INTEGRATION.md for the
 *       ~60-line glue file (`network_predict_b200(network net, float *input)`).
 *
 * Error convention: the reference has no status codes -- it prints and exits (additionally.c:1595-1614,
 * gpu.cu:58-83).  Default here is the same (message on stderr + abort()).  Hosts that prefer to recover call
 * yb_set_abort_on_error(0): failing calls then return NULL / non-zero and yb_last_error() holds the message.
 *
 * There is NO CPU fallback: every predict/forward entry point requires a CUDA device of compute capability 9.0 (H100)
 * and fails loudly without one.
 */
#ifndef YOLO2_LIGHT_B200_H
#define YOLO2_LIGHT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Numeric values are the reference's own enums so that glue code can pass `l.type` / `l.activation` through:
 * LAYER_TYPE (src/additionally.h:376-403), ACTIVATION (src/additionally.h:68-70). */
enum {
    YB_CONVOLUTIONAL = 0, YB_MAXPOOL = 3, YB_SOFTMAX = 4, YB_ROUTE = 8, YB_SHORTCUT = 13,
    YB_REGION = 21, YB_YOLO = 22, YB_UPSAMPLE = 23, YB_REORG = 24, YB_BLANK = 25
};
enum { YB_LOGISTIC = 0, YB_RELU = 1, YB_LINEAR = 3, YB_LEAKY = 7 };

/* Arithmetic used for the FP32-variant convolutions (yolov2_forward_network.c:204-211).
 *  YB_PREC_BF16_TC : bf16 operands, f32 accumulation on the wgmma tensor cores, bf16 NHWC activations (default)
 *  YB_PREC_FP32    : f32 operands and accumulation on CUDA cores, f32 activations (validation / exact nets)
 * Networks that contain XNOR layers, and every network run through an INT8 rule, always keep f32
 * activations so the integer paths see exactly the reference's inputs. */
enum { YB_PREC_BF16_TC = 0, YB_PREC_FP32 = 1 };

/* INT8 rules: what every `int quantized` argument below selects.  The reference has two INT8 forwards, and they compute
 * different things; src/main.c:199-206 runs the GPU one when built with GPU and run with -quantized.
 *  YB_QUANT_NONE (0) : no INT8 layer (network_predict_cpu / network_predict_gpu_cudnn).
 *  YB_QUANT_CPU  (1) : network_predict_quantized, src/yolov2_forward_network_quantized.c:1160.  Every other non-zero value
 *                      means this rule too.
 *      layers: conv i is INT8 iff i >= 1 and its activation is not LINEAR (:1036);
 *      input:  xq = clamp(+-127, (int16_t)(x * input_mult)) (x86 float->int16: wraps for |x * m| >= 32768);
 *      output: y = (float)clamp(+-32767, acc / 32) * (32 / (input_mult * weights_mult)) + bias, leaky as y / 10 (:474-490).
 *  YB_QUANT_GPU  (2) : network_predict_gpu_cudnn_quantized, src/yolov2_forward_network_gpu.cu:576.
 *      layers: conv i is INT8 iff the parser's l.quantized is set (forward_network_gpu_cudnn_quantized :494-507,
 *              init_gpu_int8x4 :603-611).  parse_convolutional sets it only for a cfg parsed with quantized = 1, and not
 *              for index 0, LINEAR activations, stride > 1 at index > 1, or 1x1 layers (src/additionally.c:3557-3559); the
 *              convolution whose next-but-one section is [yolo] switches it off for the rest of the net (:3996-4003).
 *              Every other convolution is a float one (an XNOR layer keeps its XNOR path, by the XNOR rule below), so a network parsed with
 *              quantized = 0 runs no INT8 layer.  yb_layer_desc.quantized carries the flag on the drop-in path.
 *      input:  v = x * input_mult rounded once, converted to int as CUDA does (truncation, saturating at +-2^31, NaN -> 0),
 *              clamped to +-127 (cuda_f32_to_int8 + max_abs, src/gpu.cu:730-739).  It agrees with the CPU rule's for
 *              |v| < 32768 and saturates above (v = 40000: +127 here, -127 there).  v <= -2^31 (and -inf) gives -127 here:
 *              max_abs read without overflow; what the reference binary makes of abs(INT_MIN) is its compiler's choice.
 *      output: y = act((float)acc * (1 / (input_mult * weights_mult)) + bias) with the exact s32 accumulator and zero
 *              padding (yolov2_forward_network_gpu.cu:184-229, :314): one rounded multiply, one rounded add, then the
 *              activation as every f32 layer computes it.  No /32, no int16 clamp.  cuDNN may fuse the multiply and the add
 *              (one rounding less); that difference cannot be checked without cuDNN.
 *      Every other layer computes what yb_network_predict computes.  Activations between layers stay f32.  With
 *      YB_PREC_FP32 the float convolutions are the reference's exact CPU arithmetic; at the default precision every float
 *      convolution the tensor cores take runs on tf32 (the reference's are cuDNN convolutions, which no fixed summation
 *      order reproduces). */
enum { YB_QUANT_NONE = 0, YB_QUANT_CPU = 1, YB_QUANT_GPU = 2 };

/* XNOR rules (yb_network_set_xnor_rule): which of the reference's two XNOR forwards an XNOR layer ([convolutional] xnor=1)
 * computes.  The default keeps every result as it was.
 *  YB_XNOR_CPU (0) : the CPU build's (forward_convolutional_layer_cpu, yolov2_forward_network.c:116-261): input bit x > 0,
 *      out-of-image taps -1, y = act((float)dot * mean + bias) with a rounded multiply and a rounded add; a layer with
 *      stride != 1 or pad != 1 is the float convolution of +-1 inputs (zero padding) and +-mean weights.
 *  YB_XNOR_GPU (1) : the GPU build's (forward_convolutional_layer_gpu_cudnn, yolov2_forward_network_gpu.cu:23-139).  With
 *      quantized = 0 it replaces network_predict_gpu_cudnn; with quantized = 2 (YB_QUANT_GPU) it completes
 *      network_predict_gpu_cudnn_quantized, whose l.quantized XNOR layers run in INT8.  quantized = 1 fails: no reference
 *      binary runs that combination.  mean is the layer's mean_arr[f].
 *    A. c % 32 == 0, any size, stride and pad: the bit GEMM.  Input bit x > 0, out-of-image taps -1, dot = 2*count - K
 *       exactly as on the CPU.  y = fmaf((float)dot, mean, bias) -- nvcc contracts the reference's `count * mean + bias` to
 *       one FFMA (gpu.cu:1981) -- then leaky as `y >= 0 ? y : 0.1f*y` (a float product), any other activation after it.
 *       A [shortcut] right behind the layer with w == out_w, h == out_h and c == out_c is folded into the GEMM
 *       (additionally.c:326-338): its output is from + v, with v the layer's leaky-only value, and neither the shortcut's
 *       activation nor any later one is applied to the sum.
 *    B. c < 32: the convolution of b(x) = x >= 0 ? +1 : -1 (note >=) and sign(w) * mean, out-of-image taps 0, as the exact
 *       integer sum s: y = act(s * mean + bias) with a rounded multiply and a rounded add.  The reference runs cuDNN there,
 *       whose summation order is not reproduced: this is the correctly rounded convolution.
 *    Leaky is the reference GPU build's `.1f * x`; relu and linear are exact; logistic is the double-precision one of
 *    every other layer, which may differ from the reference's float `1.f/(1.f+expf(-x))` in the last bit.
 *    Rejected when the engine is built, with a message: an XNOR layer with c >= 32 and c % 32 != 0 (the reference
 *    computes no convolution there); a same-shape [shortcut] behind an XNOR layer of path B or one that runs in INT8
 *    (the reference never writes its output); and one behind a path-A layer whose activation is neither leaky nor linear.
 *    Batch: the reference's bit GEMM computes image 0 of a batch only; here every image is computed as image 0 would be.
 *    Do not check this rule against a reference binary built for sm_90: there its XOR bmma becomes an AND-popcount one, so
 *    it no longer computes the XNOR count.  Non-XNOR layers compute what they compute under YB_XNOR_CPU. */
enum { YB_XNOR_CPU = 0, YB_XNOR_GPU = 1 };

/* One layer of a prepared network: the subset of the reference's `struct layer` (src/additionally.h:409-684)
 * that the forward path reads (SURVEY 8a, a13).  All pointers are host pointers owned by the caller; the
 * library copies what it needs. */
typedef struct yb_layer_desc {
    int type;                 /* YB_* layer type                                   (layer.type)        */
    int activation;           /* YB_* activation                                   (layer.activation)  */
    int batch_normalize;      /* non-zero: BN not folded yet                       (layer.batch_normalize) */
    int h, w, c;              /* input tensor                                       (layer.h/w/c)       */
    int n;                    /* conv: filters; route: #inputs; yolo/region: anchors (layer.n)          */
    int size, stride, pad;    /* conv/maxpool geometry (maxpool pad = cfg `padding`) (layer.size/stride/pad) */
    int out_h, out_w, out_c;  /* output tensor                                      (layer.out_*)       */
    int xnor;                 /* conv: BIT1-XNOR variant                            (layer.xnor)        */
    int quantized;            /* conv: parser's per-layer INT8 flag; YB_QUANT_GPU's layers (layer.quantized) */
    int index;                /* shortcut: absolute index of the `from` layer        (layer.index)       */
    int classes, coords, softmax, total;   /* yolo/region                            (layer.classes ...) */
    int reverse;              /* upsample/reorg                                      (layer.reverse)     */
    float scale;              /* upsample                                            (layer.scale)       */
    const int *input_layers;  /* route: n absolute layer indices                     (layer.input_layers) */
    const int *mask;          /* yolo: n anchor ids                                  (layer.mask)        */
    const float *anchors;     /* yolo: 2*total, region: 2*n                          (layer.biases)      */
    const float *weights;     /* conv: [n][c][size][size]                            (layer.weights)     */
    const float *biases;      /* conv: [n]                                           (layer.biases)      */
    const float *scales, *rolling_mean, *rolling_variance;   /* conv with BN: [n]                         */
    const int8_t *weights_int8;       /* conv, after quantisation: [n][c][size][size] (layer.weights_int8) */
    float weights_quant_multipler;    /*                                     (layer.weights_quant_multipler) */
    float input_quant_multipler;      /*                                     (layer.input_quant_multipler)   */
    const float *mean_arr;    /* conv xnor, after calculate_binary_weights: [n]      (layer.mean_arr)    */
} yb_layer_desc;

/* Host-side model: our equivalent of the reference's `network` (src/additionally.h:703-763). Opaque. */
typedef struct yb_network yb_network;

/* ---- errors ------------------------------------------------------------------------------------------ */
void        yb_set_abort_on_error(int on);   /* default 1 = reference behaviour (print + abort) */
const char *yb_last_error(void);

/* ---- model preparation (host, one-time) ------------------------------------------------------------ */

/* replaces parse_network_cfg(char *filename, int batch, int quantized)   src/additionally.c:3955
 * Same .cfg grammar and defaults (src/additionally.c:3423-3457, :3534-3897); batch>0 overrides the cfg's. */
yb_network *yb_parse_network_cfg(const char *filename, int batch, int quantized);

/* replaces load_weights_upto_cpu(network *net, char *filename, int cutoff)   src/additionally.c:3491
 * Same .weights format (src/additionally.c:3459-3529).  Returns 0 on success. */
int yb_load_weights_upto(yb_network *net, const char *filename, int cutoff);

/* replaces yolov2_fuse_conv_batchnorm(network net)   src/additionally.c:67 */
void yb_fuse_conv_batchnorm(yb_network *net);

/* replaces calculate_binary_weights(network net)   src/additionally.c:306  (binarize_weights :113,
 * mean_arr :188): per-filter mean |w| and sign bits for every xnor=1 convolution. */
void yb_calculate_binary_weights(yb_network *net);

/* replaces quantinization_and_get_multipliers(network net)   src/yolov2_forward_network_quantized.c:1402 */
void yb_quantinization_and_get_multipliers(yb_network *net);

/* Drop-in path: build a yb_network from layers prepared by the reference's own host code (after the
 * main.c:160-171 sequence).  dims = {batch, h, w, c}.  Arrays are copied. */
yb_network *yb_network_from_layers(const yb_layer_desc *layers, int n_layers, int batch, int h, int w, int c,
                                   int quantized);

void yb_free_network(yb_network *net);   /* free_network, src/additionally.c:2058 */

/* ---- introspection ----------------------------------------------------------------------------------- */
int  yb_network_num_layers(const yb_network *net);
/* out[0..8) = {n_layers, batch, h, w, c, inputs, outputs (last layer), input_calibration_size} */
void yb_network_dims(const yb_network *net, int *out8);
/* Fills *out with layer i; pointers alias memory owned by net (valid until yb_free_network). */
int  yb_network_layer(const yb_network *net, int i, yb_layer_desc *out);
const float *yb_network_input_calibration(const yb_network *net, int *count);
/* Change the batch size of a parsed network (set_batch_network, src/additionally.c:2038). Drops any engine. */
void yb_set_batch_network(yb_network *net, int batch);

/* ---- forward (device) -------------------------------------------------------------------------------- */

/* Select the device (cuda_set_device, src/gpu.cu:97) and the FP32-conv arithmetic for engines built later. */
int  yb_network_set_device(yb_network *net, int device);
int  yb_network_set_precision(yb_network *net, int precision /* YB_PREC_* */);
/* The XNOR rule (YB_XNOR_*) of the engines built after this call; drops the network's engines.  -1 on a bad value.
 * A network starts with the rule the environment variable YB_XNOR_RULE names when it is created (yb_parse_network_cfg,
 * yb_network_from_layers): "0" YB_XNOR_CPU, "1" YB_XNOR_GPU; unset means YB_XNOR_CPU, any other value fails the creation.
 * So a host whose networks are built by code it does not change -- the drop-in glue of a reference binary -- can run the
 * GPU build's XNOR arithmetic. */
int  yb_network_set_xnor_rule(yb_network *net, int rule /* YB_XNOR_* */);

/* replaces network_predict_cpu(network net, float *input)   src/yolov2_forward_network.c:632
 * (same slot as network_predict_gpu_cudnn, src/yolov2_forward_network_gpu.cu:547).
 * input: host, NCHW float, net.batch images of c*h*w in [0,1].  Returns the last layer's host output (owned by
 * net); every YOLO/REGION layer's host output is filled (yb_network_layer_output) so that box decoding works
 * exactly as after the reference call (additionally.c:4391-4398).  Unlike the reference's decoder the outputs
 * of ALL batch items are produced. */
float *yb_network_predict(yb_network *net, const float *input);

/* replaces network_predict_quantized(network net, float *input)   src/yolov2_forward_network_quantized.c:1160
 * INT8 rule of yolov2_forward_network_q (:1036): conv i uses the s8 x s8 -> s32 path iff i >= 1 and its
 * activation is not LINEAR; everything else as in yb_network_predict with f32 activations. */
float *yb_network_predict_quantized(yb_network *net, const float *input);

/* replaces network_predict_gpu_cudnn_quantized(network net, float *input)   src/yolov2_forward_network_gpu.cu:576
 * The YB_QUANT_GPU rule (see there); outputs as in yb_network_predict. */
float *yb_network_predict_cudnn_quantized(yb_network *net, const float *input);

/* Input pipeline on the device (SURVEY 8f row 2): replaces load_image_stb's u8 -> float/255 conversion
 * (src/additionally.c:3080-3103) + resize_image (src/additionally.c:3021-3064) + network_predict_*.
 * images_hwc: net.batch interleaved 8-bit images (HWC, net.c channels, as stbi_load returns them), all w x h.
 * The bilinear resize to the network size is bit-identical to the reference's (scalar build).  The one-size case of
 * yb_network_predict_frames_u8. */
float *yb_network_predict_image_u8(yb_network *net, const unsigned char *images_hwc, int w, int h, int quantized);

/* Letterboxing of the frame calls (off by default).  Off, every call below that resizes frames (predict_image_u8,
 * predict_frames_u8, submit_u8, submit_frames_u8, predict_device_frames, submit_device_frames) stretches each frame to the
 * network size W x H.  On, it letterboxes each frame as darknet's letterbox_image does: a w x h frame is resized
 * (resize_image, bit-identical to the reference) to its letterbox size nw x nh -- nw = W, nh = (h * W) / w when
 * (float)W / w < (float)H / h, else nh = H, nw = (w * H) / h (correct_yolo_boxes' expression, src/additionally.c:4287-4294)
 * -- and embedded at ((W - nw) / 2, (H - nh) / 2) in an input filled with 0.5.  A frame of the network's aspect ratio is
 * the same input either way.  The switch takes effect at the next call, without an engine rebuild; a submitted ticket
 * keeps the geometry it was submitted with.  The float-input calls are not affected.
 * `letter` of the detection calls still only chooses the box correction: pass letter = 1 with letterboxing on to get boxes
 * in frame coordinates (letter = 0 with it off).  With it on, a frame whose letterbox size has a side below 2 pixels (a
 * 640 x 10 frame in a 64 x 64 network) is rejected before any device work, with the frame's index and letterbox size. */
int yb_network_set_letterbox(yb_network *net, int on);

/* 1 <= nimg <= net.batch 8-bit HWC frames (net.c channels), frame b is w[b] x h[b]; each is converted and resized exactly as
 * load_image_stb + resize_image do it (src/additionally.c:3021-3103), as the reference app does per image (src/main.c:188-229),
 * or letterboxed (yb_network_set_letterbox).
 * Batch items nimg .. batch-1 are zero images.  Each frame is copied to the device on its own (frames that lie back to back
 * in host memory in one copy); the copies overlap other work only when the frames are in pinned memory (yb_alloc_pinned),
 * pageable frames work but each copy then serialises.  Rejected before any device work: nimg outside 1..net.batch, a null
 * frames / w / h array or frame, w[b] < 1 or h[b] < 1, a frame of more than INT_MAX bytes, and with letterboxing on a frame
 * whose letterbox size has a side below 2. */
float *yb_network_predict_frames_u8(yb_network *net, const unsigned char *const *frames, const int *w, const int *h,
                                    int nimg, int quantized);
/* Diagnostic: the planar float input (batch*c*h*w) the device pipeline produced for the last predict_image_u8 /
 * predict_frames_u8 / predict_device_frames call (letterboxed when yb_network_set_letterbox is on). */
int    yb_network_fetch_input(yb_network *net, int quantized, float *dst);

/* Pipelined form of the two calls above for throughput serving: yb_network_submit enqueues one batch (H2D of
 * `input` on a copy stream, the forward on the compute stream, D2H of the yolo/region tensors on a third stream)
 * and returns a ticket immediately; yb_network_collect blocks until that batch is done and points the layers'
 * host outputs at its results (valid until the ticket's slot is reused, i.e. for the next 2 submits).  Up to 3
 * batches may be in flight, so the copies of batch k+1 / k-1 overlap the compute of batch k.  `input` should be
 * pinned (yb_alloc_pinned) and must stay untouched until its ticket has been collected. */
int yb_network_submit(yb_network *net, const float *input, int quantized);
int yb_network_collect(yb_network *net, int ticket, int quantized);

/* The serving loop of the reference app (src/main.c:188-229: load_image + resize_image, network_predict*, get_network_boxes,
 * do_nms_sort) as ONE pipelined call per batch: yb_network_submit_u8 enqueues the H2D of net.batch 8-bit HWC frames (all
 * w x h) and the reference's bilinear resize on a copy stream, the forward on the compute stream and the decode + NMS of the
 * whole batch (the arithmetic of yb_network_detect) on a side stream where it runs under the NEXT batch's forward; it returns
 * a ticket at once.  yb_network_collect_detections blocks until that batch is decoded and copies back exactly its candidate
 * rows: *rows = pinned float[batch][max_rows][5 + classes] owned by the library (valid until the ticket's slot is reused, i.e.
 * for the next 2 submits), *counts = int[batch] candidates per image before the max_rows cap (max_rows <= 16384),
 * *d2h_bytes (optional) = bytes that crossed PCIe for this ticket.  Returns 5 + classes, or -1.  Up to 3 batches in flight.
 * Per batch of 16 608x608 frames that is 17.7 MB in and < 1 MB out instead of 71 MB in / 124 MB out for the raw tensors. */
int yb_network_submit_u8(yb_network *net, const unsigned char *images_hwc, int w, int h, int quantized, float thresh,
                         float nms, int relative, int letter, int max_rows);
int yb_network_collect_detections(yb_network *net, int ticket, int quantized, const float **rows, const int **counts,
                                  size_t *d2h_bytes);
/* The same serving loop for frames of different sizes and partial batches: 1 <= nimg <= net.batch frames, frame b is
 * w[b] x h[b], each resized as load_image + resize_image do it, or letterboxed (yb_network_set_letterbox, then pass
 * letter = 1), and its boxes corrected for its own size (correct_yolo_boxes src/additionally.c:4281-4315), per image as in
 * src/main.c:188-229.  Same slots, streams and ticket rules as
 * yb_network_submit_u8 (which is its one-size case); collected with yb_network_collect_detections, whose counts[b] is 0 for
 * b >= nimg.  When all nimg frames have the network size the stem reads the 8-bit frames directly.  Frames as in
 * yb_network_predict_frames_u8 (pinned memory for overlapped copies; untouched until the ticket is collected), same argument
 * checks, and max_rows in 1..16384. */
int yb_network_submit_frames_u8(yb_network *net, const unsigned char *const *frames, const int *w, const int *h, int nimg,
                                int quantized, float thresh, float nms, int relative, int letter, int max_rows);

/* Frames already in device memory: what a hardware video decoder (NV12) or a GPU JPEG decoder (planar RGB) produces, or
 * pitched RGB / BGR surfaces.  No host copy is made: the resize kernel reads each frame where it lies.  Frame b gives
 * bit-for-bit what the host calls above give for its equivalent host frame (resized input, detection tensors, rows and
 * counts), with boxes corrected for frame b's own w x h and `letter` as there:
 *   YB_FRAME_RGB         the same bytes without the row padding;
 *   YB_FRAME_BGR         each pixel's bytes reversed (the demo path's ipl_to_image + rgbgr_image, additionally.c:2915,3112);
 *   YB_FRAME_RGB_PLANAR  the HWC transpose of the three planes;
 *   YB_FRAME_NV12        the RGB frame of BT.601 limited-range fixed-point conversion (OpenCV's cvtColor
 *                        COLOR_YUV2RGB_NV12): with Y, U, V the bytes of pixel (x, y), U and V at bytes 2 * (x / 2) and
 *                        2 * (x / 2) + 1 of chroma row y / 2, yy = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128,
 *                        half = 1 << 19:  R = clamp((yy + half + 1673527 v) >> 20),
 *                        G = clamp((yy + half - 852492 v - 409993 u) >> 20), B = clamp((yy + half + 2116026 u) >> 20),
 *                        clamped to 0..255.
 *                        The opposite direction, which yb_network_submit_device_frames_draw writes with: an 8-bit R, G, B
 *                        becomes Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16, U = ((-38 R - 74 G + 112 B + 128) >> 8) + 128,
 *                        V = ((112 R - 94 G - 18 B + 128) >> 8) + 128 (BT.601 limited range, arithmetic shifts; Y in
 *                        16..235, U and V in 16..240).
 * Device frames are always resized by the kernel, also at the network size, and letterboxed like host frames when
 * yb_network_set_letterbox is on.  One format per call, 3-channel networks only. */
enum { YB_FRAME_RGB = 0, YB_FRAME_BGR = 1, YB_FRAME_RGB_PLANAR = 2, YB_FRAME_NV12 = 3 };

typedef struct yb_device_frame {
    const unsigned char *data;    /* RGB/BGR: first pixel, 3 bytes per pixel (HWC); RGB_PLANAR: the R plane; NV12: the Y plane */
    const unsigned char *chroma;  /* NV12: the interleaved U,V plane (h/2 rows, same pitch as Y); NULL for the other formats  */
    int w, h;
    int pitch;                    /* bytes from one row to the next: >= 3w (RGB/BGR), >= w (RGB_PLANAR, NV12)               */
    long long plane_stride;       /* RGB_PLANAR: bytes from the R plane to G and from G to B (>= pitch * h); ignored otherwise  */
} yb_device_frame;

/* nimg (1..net.batch) device frames of one format -> resize, forward; fills the host yolo/region outputs like
 * yb_network_predict_frames_u8 (synchronous).  Batch items nimg .. batch-1 are zero images.  yb_network_fetch_input returns
 * the resized input it made. */
float *yb_network_predict_device_frames(yb_network *net, const yb_device_frame *frames, int nimg, int format,
                                        int quantized, void *stream);
/* Pipelined form, like yb_network_submit_frames_u8: same 3 slots and ticket rules, collected with
 * yb_network_collect_detections (counts[b] = 0 for b >= nimg).
 *
 * Ordering with the caller's stream (both calls): `stream` is the cudaStream_t on which the caller produced the frames
 * (NULL = the legacy default stream).  The call records an event on `stream` and makes the engine's input stream wait on
 * it, so the frames are read only after the work the caller enqueued before the call.  After the last kernel that reads
 * the frames it records an event on the engine's input stream and makes `stream` wait on that, so work the caller enqueues
 * on `stream` after the call -- such as the decoder's next write into the same surfaces -- runs only once the engine is done
 * reading.  Neither call waits for the device before it returns (the predict call then waits for its own results).  Frames
 * written from another stream must be ordered before `stream` by the caller.
 *
 * Rejected before any device work: nimg outside 1..net.batch, a null frames array, a null data (or, for NV12, chroma)
 * pointer, w < 1 or h < 1, an odd w or h for NV12, a pitch or plane_stride below its minimum, an unknown format, a
 * network whose input does not have 3 channels, a frame whose addressed span exceeds INT_MAX bytes, with letterboxing on a
 * frame whose letterbox size has a side below 2, max_rows outside 1..16384.  Then a frame that is not device or managed memory of the network's device (host, pinned host, or another
 * GPU's memory; cudaPointerGetAttributes) is rejected. */
int yb_network_submit_device_frames(yb_network *net, const yb_device_frame *frames, int nimg, int format, int quantized,
                                    float thresh, float nms, int relative, int letter, int max_rows, void *stream);

/* The detector's drawing (test_detector, src/main.c:188-229, which draws with draw_detections_v3, main.c:80-148, and no
 * alphabet, so without text labels) into the device frames themselves.  yb_network_submit_device_frames_draw does what
 * yb_network_submit_device_frames does with relative = 1 -- same slots, tickets, argument checks, rows and counts -- and
 * then, on the engine's side stream behind the NMS of the batch, draws image b's selected detections into frame b, in place
 * and in the frame's own format.  The library writes through `data` (and `chroma`) of these frames: they must be writable
 * device memory of the network's device.  Two frames with the same `data` pointer are rejected before any device work (their
 * draws would race), and networks of more than 17395 classes (the reference's colour index, cls * 123457, would overflow).
 *
 * What is drawn, for image b, on its first min(counts[b], max_rows) post-NMS candidate rows:
 *   selection   (get_actual_detections, main.c:38-62): the best class is the first j, in class order, with prob[j] > best,
 *               best starting at thresh; a row is selected iff there is one (a probability equal to thresh is not);
 *   list order  (compare_by_lefts, main.c:65-70): ascending float x - w / 2 (NaN as +inf), equal keys by candidate position;
 *   draw order  (compare_by_probs, main.c:73-78): ascending prob[cls], equal keys by candidate position; a later detection
 *               overwrites an earlier one wherever they share pixels;
 *   geometry    (main.c:109-143): width = (int)(h * .006), at least 1; left = (int)((x - w / 2.) * frame w), right, top and
 *               bot likewise, in double, where a NaN or out-of-int value converts to INT_MIN as on x86; then left, top >= 0,
 *               right <= frame w - 1, bot <= frame h - 1; draw_box_width's `width` nested draw_box rectangles
 *               (additionally.c:2945-2988: each corner clamped into the frame, rows top and bot, columns left and right);
 *   colour      (get_color, additionally.c:3247, offset = cls * 123457 % classes): red, green, blue as floats, written as
 *               the bytes (unsigned char)(255 * c) that save_image_png (additionally.c:3226) writes;
 *   formats     RGB: those bytes; BGR: reversed; RGB_PLANAR: one per plane; NV12: each drawn pixel's Y, and the U, V pair
 *               of every 2x2 block with a drawn pixel, from the colour of the last detection in draw order that covers a
 *               pixel of the block (the RGB -> YUV rule above).  Row padding and pixels that no box covers are never written.
 * An RGB frame so drawn is byte for byte the reference's predictions.png of that frame and those rows.
 *
 * Ordering: as for yb_network_submit_device_frames, except that `stream` is made to wait on an event recorded after the
 * draw, so the work the caller enqueues on `stream` after the call (an encoder reading the frames, the decoder's next write
 * into them) sees the drawn frames.
 *
 * yb_network_collect_detections collects these tickets as any other (same rows and counts) and also copies the selected
 * list, whose bytes *d2h_bytes includes.  Then yb_network_selected_detections gives that list, valid as long as the rows:
 * *dets = pinned yb_detection[batch][max_rows] in list order, *counts = int[batch] selected detections per image (0 for
 * b >= nimg); `row` is the detection's index among the ticket's candidate rows of its image, prob = prob[cls].  It returns
 * 0, or -1 (without an error) for a ticket that is not a drawing ticket, has not been collected, or whose slot has been
 * taken by a later submit. */
typedef struct yb_detection { float x, y, w, h; float prob; int cls; int row; } yb_detection;

int yb_network_submit_device_frames_draw(yb_network *net, const yb_device_frame *frames, int nimg, int format,
                                         int quantized, float thresh, float nms, int letter, int max_rows, void *stream);
int yb_network_selected_detections(yb_network *net, int ticket, const yb_detection **dets, const int **counts);

/* Host output (NCHW for yolo, HWC-flattened for region, as the reference lays them out) of layer i after a
 * predict call; only YOLO/REGION layers (and the last layer) are kept on the host. */
const float *yb_network_layer_output(const yb_network *net, int i, int *count);

/* Device-resident variant for pipelines that already hold their images in HBM (and for the bench's `value`):
 * d_input = device pointer to net.batch NCHW float images; stream = cudaStream_t (or NULL).  Enqueues the whole
 * forward; results stay on the device until yb_network_sync_outputs(). quantized selects the INT8 rule. */
int yb_network_forward_device(yb_network *net, const void *d_input, int quantized, void *stream);
int yb_network_sync_outputs(yb_network *net, int quantized, void *stream);   /* D2H of yolo/region tensors + sync */

/* Test/diagnostic hook: copy ANY layer's activation back as NCHW float (batch-major), whatever its device
 * layout/dtype.  dst must hold batch*out_c*out_h*out_w floats (region: batch*outputs). */
int yb_network_fetch_layer(yb_network *net, int i, int quantized, float *dst);

/* replaces forward_convolutional_layer_cpu(layer l, network_state state)  src/yolov2_forward_network.c:30,
 * forward_convolutional_layer_q(layer l, network_state state)  src/yolov2_forward_network_quantized.c:527 and
 * forward_convolutional_layer_gpu_cudnn_quantized(layer l, network_state state)  src/yolov2_forward_network_gpu.cu:143.
 * Runs conv layer `i` of net alone on `input` (host NCHW, batch*c*h*w) and writes host NCHW `output`
 * (batch*n*out_h*out_w).  variant: 0 = as yb_network_predict would run it, 1 = as the quantized rule would,
 * 2 = by the YB_QUANT_GPU arithmetic, in INT8 whatever the layer's l.quantized (as that reference function does). */
int yb_forward_convolutional_layer(yb_network *net, int i, int variant, const float *input, float *output);

/* ---- multi-GPU batch extension (SURVEY 8b "Batch extension", 8e) ------------------------------------------------------
 * The reference runs one image per call on one device (src/main.c:199-219, cuda_set_device src/gpu.cu:97-102).  From the same
 * plain-C host program -- one process, no Python, no launcher -- yb_network_predict_batch runs `nimg` images (host NCHW float,
 * nimg * c*h*w) through `ngpus` replicas of the engine: contiguous shards of net.batch whole images go round-robin to the
 * replicas (pipelined per GPU like yb_network_submit), the prepared weight arena is built on the first device and reaches the
 * others by ONE ncclBroadcast at the first call (NCCL is bound at run time; without it, or for a device list with repeats,
 * peer copies -- yb_network_replication() says which), and there is no other communication.  A partial last shard is padded
 * with zero images whose results are dropped.  Results: yb_network_batch_output(net, i, &per_image) = host float[nimg][per_image]
 * for every YOLO / REGION layer and the last layer, image k bit-identical to what yb_network_predict returns for it on one GPU.
 * yb_network_set_devices chooses the devices (default 0 .. ngpus-1; repeats allowed: several replicas on one GPU). */
int yb_network_set_devices(yb_network *net, const int *devices, int ndev);
int yb_network_predict_batch(yb_network *net, const float *images, int nimg, int ngpus, int quantized);
const float *yb_network_batch_output(const yb_network *net, int i, int *per_image);
const char *yb_network_replication(const yb_network *net);   /* "nccl" | "peer-copy" | "single" | "" (not replicated yet) */

/* Weight arena of the engine (all prepared device-side weights in one allocation) -- what a multi-GPU launcher
 * broadcasts once at init (one process per GPU; the harness uses torch.distributed/NCCL on this pointer).
 * Builds the engine if needed; upload=0 allocates without uploading (non-root ranks). */
int yb_network_weight_arena(yb_network *net, int quantized, int upload, void **d_ptr, size_t *bytes);

/* Number of kernels enqueued by the last forward. */
int  yb_network_last_launches(const yb_network *net);

/* Diagnostic switches (tests): "fuse" (1: conv+shortcut fusion and route aliasing, default), "keep_counts"
 * (1: keep the raw XNOR popcounts / INT8 s32 accumulators of every integer conv), "q_index_offset".  Returns -1 for an
 * unknown name. */
int  yb_network_set_option(yb_network *net, const char *name, int value);
/* Engine facts (builds the engine if needed): "launches", "tc_layers" (convolutions on the tensor cores),
   "act_bytes" (device memory of the activation buffers), "xnor_rule" (the engine's YB_XNOR_*).  -1: unknown key. */
long yb_network_get_info(yb_network *net, int quantized, const char *key);
/* The tensor-core plan of layer `layer` (builds the engine if needed), read-only: up to n of {kernel (0 k_conv_tc,
 * 1 k_conv_tc_reg, 2 k_stem_tc, 3 k_stem_s2_tc), kind (0 bf16, 1 int8, 2 xnor, 3 tf32, 4 int8 of YB_QUANT_GPU, 5 xnor and 6 zero-padded +-1 of YB_XNOR_GPU), TW, TH, BN, BK, nt, bstat, stages,
 * sps, grid, num_work, tma_epi, jshift, out_ldc (output pixel stride, elements; 0: no NHWC output)} into fields; -1 in a
 * field that does not apply to the kernel (the stems' fixed tiles).  Returns the number written: 0 for a layer without a
 * tensor-core plan, -1 on error. */
int  yb_network_tc_plan(yb_network *net, int quantized, int layer, int *fields, int n);
/* Raw integer results of conv layer i (NCHW, batch-major) when "keep_counts" is on; returns the element count. */
int  yb_network_fetch_counts(yb_network *net, int i, int quantized, int32_t *dst, size_t count);
int  yb_network_layer_outputs(const yb_network *net, int i);   /* layer.outputs (per image) */
const char *yb_op_kind_name(int kind);
/* The engine's ops in launch order (builds the engine if needed), read-only: up to max of {layer index, op kind code, name
 * of the kernel the op launches (cudaFuncGetName; NULL for a tensor-core convolution, which launches through its plan)}.
 * Returns the number of ops, -1 on error. */
int  yb_network_op_kernels(yb_network *net, int quantized, int *layer_idx, int *op_kind, const char **name, int max);

/* Pinned host buffers for the end-to-end path (cudaHostAlloc / cudaFreeHost). */
void *yb_alloc_pinned(size_t bytes);
void  yb_free_pinned(void *p);

/* Per-op timing of one forward (CUDA events around every kernel; diagnostic, not for benchmarks).
 * Fills up to max entries: layer index, op kind code, milliseconds. Returns the number of ops. */
int yb_network_profile(yb_network *net, int quantized, const void *d_input, int *layer_idx, int *op_kind,
                       float *ms, int max);

/* ---- detection decode (host; SURVEY 8f row 1) -------------------------------------------------------- */

/* replaces get_network_boxes + do_nms_sort   src/additionally.c:4403, src/box.c:296 for batch item b.
 * out rows: {x, y, w, h, objectness, prob[classes]}; returns the number of rows written (<= max_rows).
 * Candidates with EQUAL class probability are ranked by their position in the candidate list (layer, cell, anchor), here and
 * in yb_network_detect; the reference leaves their order to qsort (box.c:311), i.e. to the C library. */
int yb_get_network_boxes(const yb_network *net, int b, int w, int h, float thresh, float nms, int relative,
                         int letter, float *out, int max_rows);

/* ---- detection decode + NMS on the device, whole batch (SURVEY 8f row 1) ------------------------------- */

/* Same arithmetic as yb_get_network_boxes / the reference (get_yolo_detections src/additionally.c:4317,
 * custom_get_region_detections :4363, correct_yolo_boxes :4281, do_nms_sort src/box.c:296), run on the yolo / region
 * tensors where the last forward left them in HBM, for every image of the batch (the reference decodes batch item 0
 * only).  rows: host float[batch][max_rows][5 + classes] = {x, y, w, h, objectness, prob[classes]} in the reference's
 * candidate order (layer, cell, anchor); suppressed / below-threshold class entries are 0 like the reference leaves
 * them.  counts[b] = number of candidates of image b; when it exceeds max_rows only the first max_rows candidates were
 * decoded and took part in the NMS (the reference has no cap: size max_rows accordingly, <= 16384).
 * Returns the row length 5 + classes, or -1. */
int yb_network_detect(yb_network *net, int quantized, int w, int h, float thresh, float nms, int relative, int letter,
                      float *rows, int max_rows, int *counts);
/* yb_network_detect for the first nimg images of the batch, image b's boxes corrected for a w[b] x h[b] frame
 * (correct_yolo_boxes src/additionally.c:4281-4315; with letter, each image's own letterbox size); counts[b] = 0 for
 * b >= nimg.  yb_network_detect is its one-size case.  Rejected before any device work: nimg outside 1..net.batch, a null w
 * / h array, w[b] < 1 or h[b] < 1, max_rows outside 1..16384. */
int yb_network_detect_frames(yb_network *net, int quantized, const int *w, const int *h, int nimg, float thresh, float nms,
                             int relative, int letter, float *rows, int max_rows, int *counts);

/* ---- INT8 input calibration (SURVEY 8f row 3) ---------------------------------------------------------- */

/* network_calibrate_cpu (src/yolov2_forward_network.c:731-831) with the forward pass and the |x| histograms of every
 * convolution's input on the GPU and entropy_calibration's KL search (src/yolov2_forward_network_quantized.c:1292-1398)
 * restated on the host.  One call = one batch of calibration images: multipliers[b * nconv + k] is what the reference
 * computes for image b at its k-th CONVOLUTIONAL layer (bin width 1/16, 4096 bins, :784).  Average over images and
 * write them as `input_calibration = m0, m1, ..., 16` into the cfg (:753-769).  Uses the network's precision setting
 * (YB_PREC_FP32 reproduces the reference's float activations); returns nconv, or -1. */
int yb_network_calibrate(yb_network *net, const float *input, float *multipliers, int max_values);
/* entropy_calibration (src/yolov2_forward_network_quantized.c:1292) on a host array: bit-identical multiplier. */
float yb_entropy_calibration(const float *src, size_t size, float bin_width, int max_bin);
/* |x| histogram of the input of layer `layer`, image `img`, after the last forward (diagnostic / tests). */
int yb_network_input_histogram(yb_network *net, int quantized, int layer, int img, float bin_width, int max_bin,
                               uint32_t *hist);

/* ---- mAP accounting (SURVEY 8f row 4) ------------------------------------------------------------------ */

/* The bookkeeping of validate_detector_map (src/additionally.c:4541-4898) on detections produced elsewhere: `rows` =
 * the concatenated rows of all images ({x, y, w, h, objectness, prob[classes]}, relative coordinates; what
 * yb_network_detect / yb_get_network_boxes return for w = h = 1, thresh .005, nms .45 as the reference uses),
 * rows_per_image[nimages]; truth[ntruth][6] = {image, class, x, y, w, h} (the label files' content, in file order).
 * Outputs: ap_per_class[classes] (11-point interpolated AP, :4848), *map_out, stats[8] = {precision, recall, F1,
 * average IoU, TP, FP, FN at thresh_calc_avg_iou (:4872-4880), number of detections}.  Returns the number of
 * (box, class) detections ranked, or -1.  The "difficult" list is not modelled. */
int yb_map_evaluate(const float *rows, const int *rows_per_image, int nimages, int classes, const float *truth, int ntruth,
                    float iou_thresh, float thresh_calc_avg_iou, double *ap_per_class, double *map_out, float *stats);

const char *yb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* YOLO2_LIGHT_B200_H */
