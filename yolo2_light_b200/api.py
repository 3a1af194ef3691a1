"""ctypes binding of ``libyolo2_light_b200.so`` -- the host-side mirror of the reference's C interface for the
forward path (same names, argument meaning and call order as ``src/main.c:160-219``):

    net = parse_network_cfg(cfg, batch, quantized)        # additionally.c:3955
    load_weights_upto_cpu(net, weights, net.n)            # additionally.c:3491
    yolov2_fuse_conv_batchnorm(net)                       # additionally.c:67
    calculate_binary_weights(net)                         # additionally.c:306
    quantinization_and_get_multipliers(net)               # yolov2_forward_network_quantized.c:1402 (if quantized)
    out = network_predict_b200(net, images)               # slot of network_predict_cpu / _gpu_cudnn
    out = network_predict_b200_quantized(net, images)     # slot of network_predict_quantized
    out = network_predict_b200_cudnn_quantized(net, images)   # slot of network_predict_gpu_cudnn_quantized

Every ``quantized`` argument selects an INT8 rule: 0 (or False) none, 1 (or True) the CPU build's, 2 the GPU build's
(YB_QUANT_NONE / YB_QUANT_CPU / YB_QUANT_GPU of the C header).

Everything heavy happens inside the shared library (CUDA, sm_90a); this module only marshals pointers.  There is
no CPU fallback: if the library is missing or no sm_90 GPU (H100) is visible the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("YB_LIB") or os.path.join(_HERE, "libyolo2_light_b200.so")   # YB_LIB: A/B builds (development)

YB_CONVOLUTIONAL, YB_MAXPOOL, YB_SOFTMAX, YB_ROUTE, YB_SHORTCUT = 0, 3, 4, 8, 13
YB_REGION, YB_YOLO, YB_UPSAMPLE, YB_REORG, YB_BLANK = 21, 22, 23, 24, 25
YB_LOGISTIC, YB_RELU, YB_LINEAR, YB_LEAKY = 0, 1, 3, 7
YB_PREC_BF16_TC, YB_PREC_FP32 = 0, 1
YB_QUANT_NONE, YB_QUANT_CPU, YB_QUANT_GPU = 0, 1, 2
YB_XNOR_CPU, YB_XNOR_GPU = 0, 1
LAYER_NAMES = {0: "CONVOLUTIONAL", 3: "MAXPOOL", 4: "SOFTMAX", 8: "ROUTE", 13: "SHORTCUT", 21: "REGION", 22: "YOLO",
               23: "UPSAMPLE", 24: "REORG", 25: "BLANK"}


class YbError(RuntimeError):
    pass


class LayerDesc(C.Structure):
    """``yb_layer_desc`` (include/yolo2_light_b200.h)."""
    _fields_ = [
        ("type", C.c_int), ("activation", C.c_int), ("batch_normalize", C.c_int),
        ("h", C.c_int), ("w", C.c_int), ("c", C.c_int), ("n", C.c_int),
        ("size", C.c_int), ("stride", C.c_int), ("pad", C.c_int),
        ("out_h", C.c_int), ("out_w", C.c_int), ("out_c", C.c_int),
        ("xnor", C.c_int), ("quantized", C.c_int), ("index", C.c_int),
        ("classes", C.c_int), ("coords", C.c_int), ("softmax", C.c_int), ("total", C.c_int),
        ("reverse", C.c_int), ("scale", C.c_float),
        ("input_layers", C.POINTER(C.c_int)), ("mask", C.POINTER(C.c_int)), ("anchors", C.POINTER(C.c_float)),
        ("weights", C.POINTER(C.c_float)), ("biases", C.POINTER(C.c_float)),
        ("scales", C.POINTER(C.c_float)), ("rolling_mean", C.POINTER(C.c_float)),
        ("rolling_variance", C.POINTER(C.c_float)),
        ("weights_int8", C.POINTER(C.c_int8)),
        ("weights_quant_multipler", C.c_float), ("input_quant_multipler", C.c_float),
        ("mean_arr", C.POINTER(C.c_float)),
    ]


class DeviceFrame(C.Structure):
    """``yb_device_frame`` (include/yolo2_light_b200.h)."""
    _fields_ = [("data", C.c_void_p), ("chroma", C.c_void_p), ("w", C.c_int), ("h", C.c_int), ("pitch", C.c_int),
                ("plane_stride", C.c_longlong)]


class Detection(C.Structure):
    """``yb_detection`` (include/yolo2_light_b200.h): one selected detection of a drawing ticket."""
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("w", C.c_float), ("h", C.c_float), ("prob", C.c_float),
                ("cls", C.c_int), ("row", C.c_int)]


# the same record as a numpy dtype
DETECTION_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("prob", "<f4"), ("cls", "<i4"),
                            ("row", "<i4")])

# ``YB_FRAME_*``: the layouts of device frames
FRAME_FORMATS = {"rgb": 0, "bgr": 1, "planar": 2, "nv12": 3}

_lib = None


def lib():
    """Load the shared library (fails loudly when it has not been built: ``python -c 'import __graft_entry__ as g;
    g.build()'`` or ``make -C yolo2_light_b200/csrc``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise YbError(f"{LIB_PATH} not built -- run __graft_entry__.build(); there is no Python/CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, ip, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float)
    sig = {
        "yb_set_abort_on_error": (None, [C.c_int]),
        "yb_last_error": (C.c_char_p, []),
        "yb_version": (C.c_char_p, []),
        "yb_parse_network_cfg": (vp, [C.c_char_p, C.c_int, C.c_int]),
        "yb_load_weights_upto": (C.c_int, [vp, C.c_char_p, C.c_int]),
        "yb_fuse_conv_batchnorm": (None, [vp]),
        "yb_calculate_binary_weights": (None, [vp]),
        "yb_quantinization_and_get_multipliers": (None, [vp]),
        "yb_network_from_layers": (vp, [C.POINTER(LayerDesc), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
        "yb_free_network": (None, [vp]),
        "yb_network_num_layers": (C.c_int, [vp]),
        "yb_network_dims": (None, [vp, ip]),
        "yb_network_layer": (C.c_int, [vp, C.c_int, C.POINTER(LayerDesc)]),
        "yb_network_layer_outputs": (C.c_int, [vp, C.c_int]),
        "yb_network_input_calibration": (fp, [vp, ip]),
        "yb_set_batch_network": (None, [vp, C.c_int]),
        "yb_network_set_device": (C.c_int, [vp, C.c_int]),
        "yb_network_set_precision": (C.c_int, [vp, C.c_int]),
        "yb_network_set_xnor_rule": (C.c_int, [vp, C.c_int]),
        "yb_network_set_option": (C.c_int, [vp, C.c_char_p, C.c_int]),
        "yb_network_set_letterbox": (C.c_int, [vp, C.c_int]),
        "yb_network_get_info": (C.c_long, [vp, C.c_int, C.c_char_p]),
        "yb_network_tc_plan": (C.c_int, [vp, C.c_int, C.c_int, ip, C.c_int]),
        "yb_network_calibrate": (C.c_int, [vp, vp, vp, C.c_int]),
        "yb_entropy_calibration": (C.c_float, [vp, C.c_size_t, C.c_float, C.c_int]),
        "yb_network_input_histogram": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, vp]),
        "yb_map_evaluate": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_float, C.c_float, vp, vp, vp]),
        "yb_network_detect": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, vp, C.c_int, vp]),
        "yb_network_submit_u8": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int]),
        "yb_network_predict_frames_u8": (fp, [vp, vp, vp, vp, C.c_int, C.c_int]),
        "yb_network_detect_frames": (C.c_int, [vp, C.c_int, vp, vp, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, vp, C.c_int, vp]),
        "yb_network_submit_frames_u8": (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int]),
        "yb_network_collect_detections": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(fp), C.POINTER(ip), C.POINTER(C.c_size_t)]),
        "yb_network_predict_device_frames": (fp, [vp, vp, C.c_int, C.c_int, C.c_int, vp]),
        "yb_network_submit_device_frames": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                                      C.c_int, C.c_int, vp]),
        "yb_network_submit_device_frames_draw": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                                           C.c_int, vp]),
        "yb_network_selected_detections": (C.c_int, [vp, C.c_int, C.POINTER(C.POINTER(Detection)), C.POINTER(ip)]),
        "yb_network_set_devices": (C.c_int, [vp, ip, C.c_int]),
        "yb_network_predict_batch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int]),
        "yb_network_batch_output": (fp, [vp, C.c_int, ip]),
        "yb_network_replication": (C.c_char_p, [vp]),
        "yb_network_predict": (fp, [vp, vp]),
        "yb_network_predict_quantized": (fp, [vp, vp]),
        "yb_network_predict_cudnn_quantized": (fp, [vp, vp]),
        "yb_network_predict_image_u8": (fp, [vp, vp, C.c_int, C.c_int, C.c_int]),
        "yb_network_fetch_input": (C.c_int, [vp, C.c_int, vp]),
        "yb_network_submit": (C.c_int, [vp, vp, C.c_int]),
        "yb_network_collect": (C.c_int, [vp, C.c_int, C.c_int]),
        "yb_network_layer_output": (fp, [vp, C.c_int, ip]),
        "yb_network_forward_device": (C.c_int, [vp, vp, C.c_int, vp]),
        "yb_network_sync_outputs": (C.c_int, [vp, C.c_int, vp]),
        "yb_network_fetch_layer": (C.c_int, [vp, C.c_int, C.c_int, vp]),
        "yb_network_fetch_counts": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_size_t]),
        "yb_forward_convolutional_layer": (C.c_int, [vp, C.c_int, C.c_int, vp, vp]),
        "yb_network_weight_arena": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(vp), C.POINTER(C.c_size_t)]),
        "yb_network_last_launches": (C.c_int, [vp]),
        "yb_network_profile": (C.c_int, [vp, C.c_int, vp, ip, ip, fp, C.c_int]),
        "yb_op_kind_name": (C.c_char_p, [C.c_int]),
        "yb_network_op_kernels": (C.c_int, [vp, C.c_int, ip, ip, C.POINTER(C.c_char_p), C.c_int]),
        "yb_get_network_boxes": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int,
                                           vp, C.c_int]),
        "yb_alloc_pinned": (vp, [C.c_size_t]),
        "yb_free_pinned": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        if "YB_LIB" in os.environ and not hasattr(L, name):
            continue                 # an older A/B build may lack the newest entry points
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args
    L.yb_set_abort_on_error(0)   # Python hosts get exceptions instead of abort()
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "yb_set_abort_on_error", "yb_last_error", "yb_version", "yb_parse_network_cfg", "yb_load_weights_upto",
    "yb_fuse_conv_batchnorm", "yb_calculate_binary_weights", "yb_quantinization_and_get_multipliers",
    "yb_network_from_layers", "yb_free_network", "yb_network_num_layers", "yb_network_dims", "yb_network_layer",
    "yb_network_layer_outputs", "yb_network_input_calibration", "yb_set_batch_network", "yb_network_set_device",
    "yb_network_set_precision", "yb_network_set_xnor_rule", "yb_network_set_option", "yb_network_get_info", "yb_network_tc_plan", "yb_network_detect", "yb_network_calibrate", "yb_entropy_calibration",
    "yb_network_input_histogram", "yb_map_evaluate", "yb_network_predict", "yb_network_predict_quantized",
    "yb_network_predict_cudnn_quantized",
    "yb_network_predict_image_u8", "yb_network_fetch_input", "yb_network_submit", "yb_network_collect", "yb_network_layer_output", "yb_network_forward_device", "yb_network_sync_outputs", "yb_network_fetch_layer",
    "yb_network_fetch_counts", "yb_forward_convolutional_layer", "yb_network_weight_arena",
    "yb_network_last_launches", "yb_network_profile", "yb_op_kind_name", "yb_network_op_kernels", "yb_get_network_boxes", "yb_alloc_pinned",
    "yb_free_pinned", "yb_network_submit_u8", "yb_network_collect_detections", "yb_network_set_devices",
    "yb_network_predict_batch", "yb_network_batch_output", "yb_network_replication", "yb_network_predict_frames_u8",
    "yb_network_detect_frames", "yb_network_submit_frames_u8", "yb_network_predict_device_frames",
    "yb_network_submit_device_frames", "yb_network_set_letterbox", "yb_network_submit_device_frames_draw",
    "yb_network_selected_detections",
]


TC_PLAN_FIELDS = ("kernel", "kind", "TW", "TH", "BN", "BK", "nt", "bstat", "stages", "sps", "grid", "num_work", "tma_epi",
                  "jshift", "out_ldc")
TC_PLAN_KERNELS = ("k_conv_tc", "k_conv_tc_reg", "k_stem_tc", "k_stem_s2_tc")
TC_PLAN_KINDS = ("bf16", "s8", "xnor", "tf32", "s8_gpu", "xnor_gpu", "pm1z_gpu")


def _check(ok: bool):
    if not ok:
        raise YbError(lib().yb_last_error().decode(errors="replace"))


def _np(ptr, count, dtype):
    if not ptr or count <= 0:
        return None
    return np.ctypeslib.as_array(ptr, shape=(count,)).view(dtype)


class Network:
    """Handle on a ``yb_network`` (the reference's ``network``)."""

    def __init__(self, handle: int):
        self._h = C.c_void_p(handle)
        self._refresh()

    def _refresh(self):
        d = (C.c_int * 8)()
        lib().yb_network_dims(self._h, d)
        self.n, self.batch, self.h, self.w, self.c, self.inputs, self.outputs, self.input_calibration_size = list(d)

    def __del__(self):
        try:
            if self._h:
                lib().yb_free_network(self._h)
                self._h = None
        except Exception:
            pass

    # -- introspection -------------------------------------------------------------------------------
    def layer_desc(self, i: int) -> LayerDesc:
        d = LayerDesc()
        _check(lib().yb_network_layer(self._h, i, C.byref(d)) == 0)
        return d

    def layer(self, i: int) -> dict:
        d = self.layer_desc(i)
        out = {k: getattr(d, k) for k, _ in LayerDesc._fields_ if not isinstance(getattr(d, k), C._Pointer)}
        out["outputs"] = lib().yb_network_layer_outputs(self._h, i)
        out["type_name"] = LAYER_NAMES.get(d.type, str(d.type))
        nw = d.n * d.c * d.size * d.size
        if d.type == YB_CONVOLUTIONAL:
            out["weights"] = _np(d.weights, nw, np.float32)
            out["biases"] = _np(d.biases, d.n, np.float32)
            out["scales"] = _np(d.scales, d.n, np.float32)
            out["rolling_mean"] = _np(d.rolling_mean, d.n, np.float32)
            out["rolling_variance"] = _np(d.rolling_variance, d.n, np.float32)
            out["weights_int8"] = _np(d.weights_int8, nw, np.int8)
            out["mean_arr"] = _np(d.mean_arr, d.n, np.float32)
        elif d.type == YB_ROUTE:
            out["input_layers"] = _np(d.input_layers, d.n, np.int32)
        elif d.type == YB_YOLO:
            out["mask"] = _np(d.mask, d.n, np.int32)
            out["anchors"] = _np(d.anchors, 2 * d.total, np.float32)
        elif d.type == YB_REGION:
            out["anchors"] = _np(d.anchors, 2 * d.n, np.float32)
        return out

    @property
    def layers(self) -> List[dict]:
        return [self.layer(i) for i in range(self.n)]

    def input_calibration(self) -> np.ndarray:
        cnt = C.c_int()
        p = lib().yb_network_input_calibration(self._h, C.byref(cnt))
        a = _np(p, cnt.value, np.float32)
        return np.zeros(0, np.float32) if a is None else a.copy()

    # -- configuration -------------------------------------------------------------------------------
    def set_batch(self, batch: int):
        lib().yb_set_batch_network(self._h, batch)
        self._refresh()

    def set_device(self, device: int):
        _check(lib().yb_network_set_device(self._h, device) == 0)

    def set_precision(self, precision: int):
        _check(lib().yb_network_set_precision(self._h, precision) == 0)

    def set_xnor_rule(self, rule: int):
        """The XNOR arithmetic of the engines built after this call (``yb_network_set_xnor_rule``): ``YB_XNOR_CPU``
        (default), the reference CPU build's, or ``YB_XNOR_GPU``, its GPU build's."""
        _check(lib().yb_network_set_xnor_rule(self._h, rule) == 0)

    def set_option(self, name: str, value: int):
        _check(lib().yb_network_set_option(self._h, name.encode(), value) == 0)

    def set_letterbox(self, on: bool):
        """Letterbox frames instead of stretching them in every frame call (``yb_network_set_letterbox``); pass
        ``letter=1`` to the detection calls to get boxes in frame coordinates.  Takes effect at the next call."""
        _check(lib().yb_network_set_letterbox(self._h, int(bool(on))) == 0)

    def get_info(self, key: str, quantized: bool = False) -> int:
        return int(lib().yb_network_get_info(self._h, int(quantized), key.encode()))

    def tc_plan(self, i: int, quantized: bool = False) -> dict:
        """The tensor-core plan of layer i (see yb_network_tc_plan): kernel and kind by name, the tile parameters as ints
        (-1: does not apply to that kernel); {} for a layer without one."""
        f = (C.c_int * len(TC_PLAN_FIELDS))()
        r = lib().yb_network_tc_plan(self._h, int(quantized), i, f, len(f))
        _check(r >= 0)
        if r == 0:
            return {}
        d = dict(zip(TC_PLAN_FIELDS, list(f)[:r]))
        d["kernel"] = TC_PLAN_KERNELS[d["kernel"]]
        d["kind"] = TC_PLAN_KINDS[d["kind"]]
        return d

    # -- forward -------------------------------------------------------------------------------------
    def _out_shape(self, i: int):
        d = self.layer_desc(i)
        if d.type == YB_REGION:
            return (self.batch, -1)
        return (self.batch, d.out_c, d.out_h, d.out_w)

    def predict(self, images: np.ndarray, quantized: bool = False) -> np.ndarray:
        x = np.ascontiguousarray(images, dtype=np.float32)
        if x.size != self.batch * self.c * self.h * self.w:
            raise YbError(f"input has {x.size} floats, network wants batch {self.batch} x {self.c}x{self.h}x{self.w}")
        rule = int(quantized)
        f = (lib().yb_network_predict_cudnn_quantized if rule == YB_QUANT_GPU else
             lib().yb_network_predict_quantized if rule else lib().yb_network_predict)
        p = f(self._h, x.ctypes.data_as(C.c_void_p))
        _check(bool(p))
        return self.layer_output(self.n - 1)

    def predict_image_u8(self, images_hwc: np.ndarray, quantized: bool = False) -> np.ndarray:
        """u8 HWC images [batch, h, w, c] of any size -> device-side /255 + bilinear resize (the reference's
        load_image_stb + resize_image) -> forward."""
        x = np.ascontiguousarray(images_hwc, dtype=np.uint8)
        if x.ndim != 4 or x.shape[0] != self.batch or x.shape[3] != self.c:
            raise YbError(f"predict_image_u8 wants [batch={self.batch}, h, w, c={self.c}] uint8, got {x.shape}")
        p = lib().yb_network_predict_image_u8(self._h, x.ctypes.data_as(C.c_void_p), x.shape[2], x.shape[1], int(quantized))
        _check(bool(p))
        return self.layer_output(self.n - 1)

    def _frames(self, frames, fn: str):
        """1..batch uint8 [h_i, w_i, c] arrays -> (keep-alive list, pointer array, w array, h array)."""
        frames = list(frames)
        if not 1 <= len(frames) <= self.batch:
            raise YbError(f"{fn}: {len(frames)} frames, the network takes 1..{self.batch}")
        keep = []
        for k, f in enumerate(frames):
            if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != self.c:
                raise YbError(f"{fn}: frame {k} must be a uint8 [h, w, c={self.c}] array, got "
                              f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', None)}")
            keep.append(np.ascontiguousarray(f))
        ptrs = (C.c_void_p * len(keep))(*[f.ctypes.data for f in keep])
        ws = (C.c_int * len(keep))(*[f.shape[1] for f in keep])
        hs = (C.c_int * len(keep))(*[f.shape[0] for f in keep])
        return keep, ptrs, ws, hs

    def predict_frames_u8(self, frames, quantized: bool = False) -> np.ndarray:
        """1..batch uint8 [h_i, w_i, c] frames, each of its own size -> the reference's per-image load + resize on the device ->
        forward (``yb_network_predict_frames_u8``).  Batch items past the frames are zero images."""
        keep, ptrs, ws, hs = self._frames(frames, "predict_frames_u8")
        p = lib().yb_network_predict_frames_u8(self._h, ptrs, ws, hs, len(keep), int(quantized))
        _check(bool(p))
        return self.layer_output(self.n - 1)

    def fetch_input(self, quantized: bool = False) -> np.ndarray:
        dst = np.empty((self.batch, self.c, self.h, self.w), np.float32)
        _check(lib().yb_network_fetch_input(self._h, int(quantized), dst.ctypes.data_as(C.c_void_p)) == 0)
        return dst

    def submit(self, images: np.ndarray, quantized: bool = False) -> int:
        """Pipelined predict: enqueue one batch, returns a ticket (see yb_network_submit)."""
        x = images if (isinstance(images, np.ndarray) and images.dtype == np.float32 and images.flags.c_contiguous) \
            else np.ascontiguousarray(images, dtype=np.float32)
        if x.size != self.batch * self.c * self.h * self.w:
            raise YbError("submit: wrong input size")
        self._inflight = getattr(self, "_inflight", {})
        t = lib().yb_network_submit(self._h, x.ctypes.data_as(C.c_void_p), int(quantized))
        _check(t >= 0)
        self._inflight[t] = x   # keep the host buffer alive until collected
        return t

    def collect(self, ticket: int, quantized: bool = False) -> dict:
        _check(lib().yb_network_collect(self._h, ticket, int(quantized)) == 0)
        getattr(self, "_inflight", {}).pop(ticket, None)
        return self.detection_outputs()

    def submit_u8(self, images_hwc: np.ndarray, thresh: float, nms: float = 0.45, relative: int = 1, letter: int = 0,
                  max_rows: int = 2048, quantized: bool = False) -> int:
        """Pipelined u8 frames -> detections (``yb_network_submit_u8``): images_hwc uint8 [batch, h, w, c]."""
        x = images_hwc if (isinstance(images_hwc, np.ndarray) and images_hwc.dtype == np.uint8 and images_hwc.flags.c_contiguous) \
            else np.ascontiguousarray(images_hwc, dtype=np.uint8)
        if x.ndim != 4 or x.shape[0] != self.batch or x.shape[3] != self.c:
            raise YbError("submit_u8: expected uint8 [batch, h, w, c]")
        self._inflight = getattr(self, "_inflight", {})
        t = lib().yb_network_submit_u8(self._h, x.ctypes.data_as(C.c_void_p), int(x.shape[2]), int(x.shape[1]), int(quantized),
                                       thresh, nms, relative, letter, max_rows)
        _check(t >= 0)
        self._inflight[("u8", t)] = (x, max_rows, self.batch)
        return t

    def submit_frames_u8(self, frames, thresh: float, nms: float = 0.45, relative: int = 1, letter: int = 0,
                         max_rows: int = 2048, quantized: bool = False) -> int:
        """Pipelined frames of any sizes -> detections (``yb_network_submit_frames_u8``): 1..batch uint8 [h_i, w_i, c]
        arrays; each image's boxes are corrected for its own frame size.  Returns a ticket for collect_detections."""
        keep, ptrs, ws, hs = self._frames(frames, "submit_frames_u8")
        self._inflight = getattr(self, "_inflight", {})
        t = lib().yb_network_submit_frames_u8(self._h, ptrs, ws, hs, len(keep), int(quantized), thresh, nms, relative, letter,
                                              max_rows)
        _check(t >= 0)
        self._inflight[("u8", t)] = (keep, max_rows, len(keep))
        return t

    def _device_frames(self, frames, fmt: str, fn: str):
        """1..batch device frames of format `fmt` -> (keep-alive list, yb_device_frame array, YB_FRAME_* value).

        Each frame is an object with a ``__cuda_array_interface__`` of typestr ``|u1`` (a torch CUDA tensor, a CuPy array,
        ...): rgb / bgr ``(h, w, 3)`` with strides ``(pitch, 3, 1)``; planar ``(3, h, w)`` with strides
        ``(plane, pitch, 1)``; nv12 one ``(3h/2, w)`` array with strides ``(pitch, 1)`` (the chroma plane starts at row h),
        or a ``(Y (h, w), UV (h/2, w))`` pair with the same pitch."""
        if fmt not in FRAME_FORMATS:
            raise YbError(f"{fn}: unknown format {fmt!r}, expected one of {', '.join(FRAME_FORMATS)}")
        frames = list(frames)
        if not 1 <= len(frames) <= self.batch:
            raise YbError(f"{fn}: {len(frames)} frames, the network takes 1..{self.batch}")

        def view(obj, k, what, ndim, inner):
            """(pointer, shape, strides) of a uint8 array of rank ndim whose trailing strides are `inner`."""
            cai = getattr(obj, "__cuda_array_interface__", None)
            if not isinstance(cai, dict):
                raise YbError(f"{fn}: frame {k} must expose __cuda_array_interface__ (a device array), got "
                              f"{type(obj).__name__}")
            shape = tuple(int(s) for s in cai.get("shape", ()))
            if cai.get("typestr") != "|u1" or len(shape) != ndim:
                raise YbError(f"{fn}: frame {k} must be a uint8 {what} array, got typestr {cai.get('typestr')!r} "
                              f"shape {shape}")
            strides = cai.get("strides")
            if strides is None:   # C-contiguous
                strides, acc = [], 1
                for s in reversed(shape):
                    strides.insert(0, acc)
                    acc *= s
            strides = tuple(int(s) for s in strides)
            if strides[ndim - len(inner):] != inner or not 0 < strides[0] < 2 ** 31 or (ndim == 3 and not 0 < strides[1] < 2 ** 31):
                raise YbError(f"{fn}: frame {k} must be a uint8 {what} array, got shape {shape} strides {strides}")
            return int(cai["data"][0]), shape, strides

        F = FRAME_FORMATS[fmt]
        arr = (DeviceFrame * len(frames))()
        for k, f in enumerate(frames):
            d = arr[k]
            if fmt in ("rgb", "bgr"):
                p, (h, w, c), (pitch, _, _) = view(f, k, "[h, w, 3] (strides (pitch, 3, 1))", 3, (3, 1))
                if c != 3:
                    raise YbError(f"{fn}: frame {k} must be a uint8 [h, w, 3] (strides (pitch, 3, 1)) array, got shape {(h, w, c)}")
                d.data, d.w, d.h, d.pitch = p, w, h, pitch
            elif fmt == "planar":
                p, (c, h, w), (plane, pitch, _) = view(f, k, "[3, h, w] (strides (plane, pitch, 1))", 3, (1,))
                if c != 3:
                    raise YbError(f"{fn}: frame {k} must be a uint8 [3, h, w] (strides (plane, pitch, 1)) array, got shape "
                                  f"{(c, h, w)}")
                d.data, d.w, d.h, d.pitch, d.plane_stride = p, w, h, pitch, plane
            elif isinstance(f, (tuple, list)):
                if len(f) != 2:
                    raise YbError(f"{fn}: frame {k}: an nv12 pair is (Y [h, w], UV [h/2, w]), got {len(f)} arrays")
                py, (h, w), (pitch, _) = view(f[0], k, "Y [h, w] (strides (pitch, 1))", 2, (1,))
                pc, (hc, wc), (pitch_c, _) = view(f[1], k, "UV [h/2, w] (strides (pitch, 1))", 2, (1,))
                if 2 * hc != h or wc != w or (hc > 1 and pitch_c != pitch):   # one UV row: its pitch is never used
                    raise YbError(f"{fn}: frame {k}: UV plane {(hc, wc)} with pitch {pitch_c} does not match Y plane {(h, w)} "
                                  f"with pitch {pitch} (UV must be [h/2, w] with the same pitch)")
                d.data, d.chroma, d.w, d.h, d.pitch = py, pc, w, h, pitch
            else:
                p, (rows, w), (pitch, _) = view(f, k, "[3h/2, w] (strides (pitch, 1))", 2, (1,))
                if rows % 3:
                    raise YbError(f"{fn}: frame {k}: an nv12 array has 3h/2 rows, got {rows}")
                h = rows // 3 * 2
                d.data, d.chroma, d.w, d.h, d.pitch = p, p + h * pitch, w, h, pitch
        return frames, arr, F

    def predict_device_frames(self, frames, fmt: str = "rgb", quantized: bool = False, stream: Optional[int] = None):
        """1..batch frames in device memory of one format (see ``_device_frames``) -> the reference's per-image resize on the
        device -> forward (``yb_network_predict_device_frames``).  `stream`: the integer cudaStream_t the frames were written
        on (``torch.cuda.current_stream().cuda_stream``), None for the legacy default stream."""
        keep, arr, F = self._device_frames(frames, fmt, "predict_device_frames")
        p = lib().yb_network_predict_device_frames(self._h, arr, len(keep), F, int(quantized), C.c_void_p(stream or 0))
        _check(bool(p))
        return self.layer_output(self.n - 1)

    def submit_device_frames(self, frames, thresh: float, fmt: str = "rgb", nms: float = 0.45, relative: int = 1,
                             letter: int = 0, max_rows: int = 2048, quantized: bool = False,
                             stream: Optional[int] = None) -> int:
        """Pipelined device frames -> detections (``yb_network_submit_device_frames``); frames and `stream` as in
        predict_device_frames.  The frame objects are kept referenced until the ticket is collected with
        collect_detections; the stream ordering rules of the C call say when their memory may be rewritten."""
        keep, arr, F = self._device_frames(frames, fmt, "submit_device_frames")
        self._inflight = getattr(self, "_inflight", {})
        t = lib().yb_network_submit_device_frames(self._h, arr, len(keep), F, int(quantized), thresh, nms, relative, letter,
                                                  max_rows, C.c_void_p(stream or 0))
        _check(t >= 0)
        self._inflight[("u8", t)] = (keep, max_rows, len(keep))
        return t

    def submit_device_frames_draw(self, frames, thresh: float, fmt: str = "rgb", nms: float = 0.45, letter: int = 0,
                                  max_rows: int = 2048, quantized: bool = False, stream: Optional[int] = None) -> int:
        """submit_device_frames with relative boxes, which then draws each image's selected detections into its frame, in
        place, as the reference's test_detector draws them (``yb_network_submit_device_frames_draw``).  The frames must be
        writable device memory and distinct; `stream` waits for the draw.  Collect with collect_detections, then read the
        selected list with selected_detections."""
        keep, arr, F = self._device_frames(frames, fmt, "submit_device_frames_draw")
        self._inflight = getattr(self, "_inflight", {})
        t = lib().yb_network_submit_device_frames_draw(self._h, arr, len(keep), F, int(quantized), thresh, nms, letter,
                                                       max_rows, C.c_void_p(stream or 0))
        _check(t >= 0)
        self._inflight[("u8", t)] = (keep, max_rows, len(keep))
        return t

    def selected_detections(self, ticket: int):
        """The selected list of a collected drawing ticket (``yb_network_selected_detections``): one DETECTION_DTYPE array
        per image of the ticket, in list order (ascending left edge); None for any other ticket."""
        dets, counts = C.POINTER(Detection)(), C.POINTER(C.c_int)()
        if lib().yb_network_selected_detections(self._h, ticket, C.byref(dets), C.byref(counts)) != 0:
            return None
        max_rows, nimg = getattr(self, "_collected", {})[ticket]
        cnt = np.ctypeslib.as_array(counts, shape=(self.batch,))
        buf = (C.c_char * (self.batch * max_rows * DETECTION_DTYPE.itemsize)).from_address(C.addressof(dets.contents))
        alld = np.frombuffer(buf, DETECTION_DTYPE).reshape(self.batch, max_rows)
        return [alld[b, :int(cnt[b])].copy() for b in range(nimg)]

    def collect_detections(self, ticket: int, quantized: bool = False, copy: bool = True):
        """Returns (list of [n_b, 5 + classes] arrays, counts int32, bytes moved device -> host) for the ticket's images:
        batch of them for submit_u8, nimg for submit_frames_u8 and submit_device_frames."""
        rows, counts, moved = C.POINTER(C.c_float)(), C.POINTER(C.c_int)(), C.c_size_t()
        stride = lib().yb_network_collect_detections(self._h, ticket, int(quantized), C.byref(rows), C.byref(counts), C.byref(moved))
        _check(stride > 0)
        _, max_rows, nimg = getattr(self, "_inflight", {}).pop(("u8", ticket), (None, None, None))
        if max_rows is None:
            raise YbError("collect_detections: unknown ticket")
        self._collected = getattr(self, "_collected", {})
        self._collected[ticket] = (max_rows, nimg)
        cnt = np.ctypeslib.as_array(counts, shape=(self.batch,))[:nimg].copy()
        allrows = np.ctypeslib.as_array(rows, shape=(self.batch, max_rows, stride))
        out = [allrows[b, :min(int(cnt[b]), max_rows)] for b in range(nimg)]
        if copy:
            out = [o.copy() for o in out]
        return out, cnt, int(moved.value)

    def set_devices(self, devices) -> None:
        arr = (C.c_int * len(devices))(*devices)
        _check(lib().yb_network_set_devices(self._h, arr, len(devices)) == 0)

    def predict_batch(self, images: np.ndarray, ngpus: int, quantized: bool = False) -> dict:
        """``yb_network_predict_batch``: any number of images over `ngpus` engine replicas of this process."""
        x = np.ascontiguousarray(images, dtype=np.float32)
        nimg = x.shape[0]
        if x.size != nimg * self.c * self.h * self.w:
            raise YbError("predict_batch: wrong input size")
        _check(lib().yb_network_predict_batch(self._h, x.ctypes.data_as(C.c_void_p), nimg, ngpus, int(quantized)) == 0)
        out = {}
        for i in range(self.n):
            per = C.c_int()
            p = lib().yb_network_batch_output(self._h, i, C.byref(per))
            if p:
                out[i] = _np(p, nimg * per.value, np.float32).reshape(nimg, -1).copy()
        return out

    def replication(self) -> str:
        return lib().yb_network_replication(self._h).decode()

    def layer_output(self, i: int) -> np.ndarray:
        """Host output of a YOLO / REGION / last layer after predict (view on pinned memory; copy to keep)."""
        cnt = C.c_int()
        p = lib().yb_network_layer_output(self._h, i, C.byref(cnt))
        if not p:
            raise YbError(f"layer {i} has no host output (only yolo/region/last layers do); use fetch_layer")
        return _np(p, cnt.value, np.float32).reshape(self._out_shape(i))

    def detection_outputs(self) -> dict:
        out = {}
        for i in range(self.n):
            t = self.layer_desc(i).type
            if t in (YB_YOLO, YB_REGION):
                out[i] = self.layer_output(i)
        return out

    def fetch_layer(self, i: int, quantized: bool = False) -> np.ndarray:
        d = self.layer_desc(i)
        count = lib().yb_network_layer_outputs(self._h, i) * self.batch
        dst = np.empty(count, np.float32)
        _check(lib().yb_network_fetch_layer(self._h, i, int(quantized), dst.ctypes.data_as(C.c_void_p)) == 0)
        return dst.reshape(self._out_shape(i))

    def fetch_counts(self, i: int, quantized: bool = False) -> np.ndarray:
        d = self.layer_desc(i)
        count = self.batch * d.n * d.out_h * d.out_w
        dst = np.empty(count, np.int32)
        r = lib().yb_network_fetch_counts(self._h, i, int(quantized), dst.ctypes.data_as(C.c_void_p), count)
        _check(r == count)
        return dst.reshape(self.batch, d.n, d.out_h, d.out_w)

    def forward_convolutional_layer(self, i: int, x: np.ndarray, variant: int = 0) -> np.ndarray:
        d = self.layer_desc(i)
        x = np.ascontiguousarray(x, dtype=np.float32)
        assert x.size == self.batch * d.c * d.h * d.w
        out = np.empty((self.batch, d.n, d.out_h, d.out_w), np.float32)
        _check(lib().yb_forward_convolutional_layer(self._h, i, variant, x.ctypes.data_as(C.c_void_p),
                                                    out.ctypes.data_as(C.c_void_p)) == 0)
        return out

    def forward_device(self, d_input_ptr: int, quantized: bool = False, stream: int = 0):
        _check(lib().yb_network_forward_device(self._h, C.c_void_p(d_input_ptr), int(quantized),
                                               C.c_void_p(stream)) == 0)

    def sync_outputs(self, quantized: bool = False, stream: int = 0):
        _check(lib().yb_network_sync_outputs(self._h, int(quantized), C.c_void_p(stream)) == 0)

    def weight_arena(self, quantized: bool = False, upload: bool = True):
        ptr, size = C.c_void_p(), C.c_size_t()
        _check(lib().yb_network_weight_arena(self._h, int(quantized), int(upload), C.byref(ptr), C.byref(size)) == 0)
        return ptr.value, size.value

    def last_launches(self) -> int:
        return lib().yb_network_last_launches(self._h)

    def profile(self, quantized: bool = False, d_input_ptr: int = 0):
        n = 4096
        li, kk, ms = (C.c_int * n)(), (C.c_int * n)(), (C.c_float * n)()
        r = lib().yb_network_profile(self._h, int(quantized), C.c_void_p(d_input_ptr), li, kk, ms, n)
        _check(r >= 0)
        return [(li[i], lib().yb_op_kind_name(kk[i]).decode(), ms[i]) for i in range(min(r, n))]

    def op_kernels(self, quantized: bool = False):
        """The engine's ops in launch order: (layer, op kind, kernel name), the name as cudaFuncGetName gives it (None for
        an op that launches through a tensor-core plan); layer -1 is the input conversion."""
        n = lib().yb_network_op_kernels(self._h, int(quantized), None, None, None, 0)
        _check(n >= 0)
        li, kk, nm = (C.c_int * max(n, 1))(), (C.c_int * max(n, 1))(), (C.c_char_p * max(n, 1))()
        _check(lib().yb_network_op_kernels(self._h, int(quantized), li, kk, nm, n) == n)
        return [(li[i], lib().yb_op_kind_name(kk[i]).decode(), nm[i].decode() if nm[i] else None) for i in range(n)]

    def get_network_boxes(self, b: int, w: int, h: int, thresh: float, nms: float = 0.0, relative: int = 1,
                          letter: int = 0, max_rows: int = 200000) -> np.ndarray:
        classes = 0
        for i in range(self.n):
            d = self.layer_desc(i)
            if d.type in (YB_YOLO, YB_REGION):
                classes = d.classes
        out = np.zeros((max_rows, 5 + classes), np.float32)
        r = lib().yb_get_network_boxes(self._h, b, w, h, thresh, nms, relative, letter,
                                       out.ctypes.data_as(C.c_void_p), max_rows)
        _check(r >= 0)
        return out[:min(r, max_rows)]


    def calibrate(self, images: np.ndarray) -> np.ndarray:
        """INT8 input calibration of one image batch (``yb_network_calibrate``): float32[batch, nconv] multipliers."""
        x = np.ascontiguousarray(images, dtype=np.float32)
        if x.size != self.batch * self.c * self.h * self.w:
            raise YbError(f"calibrate: expected {self.batch}x{self.c}x{self.h}x{self.w} floats, got {x.size}")
        nconv = sum(1 for i in range(self.n) if self.layer_desc(i).type == YB_CONVOLUTIONAL)
        out = np.zeros((self.batch, nconv), np.float32)
        r = lib().yb_network_calibrate(self._h, x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), out.size)
        _check(r == nconv)
        return out

    def input_histogram(self, layer: int, img: int = 0, bin_width: float = 1.0 / 16, max_bin: int = 4096,
                        quantized: bool = False) -> np.ndarray:
        h = np.zeros(max_bin, np.uint32)
        _check(lib().yb_network_input_histogram(self._h, int(quantized), layer, img, bin_width, max_bin,
                                                h.ctypes.data_as(C.c_void_p)) == 0)
        return h

    def detect(self, w: int, h: int, thresh: float, nms: float = 0.45, relative: int = 1, letter: int = 0,
               max_rows: int = 1024, quantized: bool = False):
        """Decode + NMS of the whole batch on the device (``yb_network_detect``).  Returns a list (one entry per image)
        of float32 arrays [candidates, 5 + classes] and the raw candidate counts."""
        classes = 0
        for i in range(self.n):
            d = self.layer_desc(i)
            if d.type in (YB_YOLO, YB_REGION):
                classes = d.classes
        rows = np.zeros((self.batch, max_rows, 5 + classes), np.float32)
        counts = np.zeros(self.batch, np.int32)
        r = lib().yb_network_detect(self._h, int(quantized), w, h, thresh, nms, relative, letter,
                                    rows.ctypes.data_as(C.c_void_p), max_rows, counts.ctypes.data_as(C.c_void_p))
        _check(r == 5 + classes)
        return [rows[b, :min(int(counts[b]), max_rows)] for b in range(self.batch)], counts

    def detect_frames(self, sizes, thresh: float, nms: float = 0.45, relative: int = 1, letter: int = 0,
                      max_rows: int = 1024, quantized: bool = False):
        """``yb_network_detect_frames``: decode + NMS of the first len(sizes) images on the device, image b's boxes corrected
        for a frame of sizes[b] = (w, h).  Returns one [candidates, 5 + classes] array per image and counts int32[nimg]."""
        sizes = [(int(w), int(h)) for w, h in sizes]
        classes = max((self.layer_desc(i).classes for i in range(self.n) if self.layer_desc(i).type in (YB_YOLO, YB_REGION)),
                      default=0)
        nimg = len(sizes)
        ws = (C.c_int * max(nimg, 1))(*[w for w, _ in sizes])
        hs = (C.c_int * max(nimg, 1))(*[h for _, h in sizes])
        rows = np.zeros((self.batch, max(max_rows, 1), 5 + classes), np.float32)
        counts = np.zeros(self.batch, np.int32)
        r = lib().yb_network_detect_frames(self._h, int(quantized), ws, hs, nimg, thresh, nms, relative, letter,
                                           rows.ctypes.data_as(C.c_void_p), max_rows, counts.ctypes.data_as(C.c_void_p))
        _check(r == 5 + classes)
        return [rows[b, :min(int(counts[b]), max_rows)] for b in range(nimg)], counts[:nimg].copy()


def map_evaluate(rows_per_image_list, truth: np.ndarray, classes: int, iou_thresh: float = 0.5,
                 thresh_calc_avg_iou: float = 0.24):
    """``yb_map_evaluate``: rows_per_image_list = one [n_i, 5 + classes] array per image (relative coordinates),
    truth = float32 [ntruth, 6] {image, class, x, y, w, h}.  Returns (mAP, ap_per_class, stats dict)."""
    rows = [np.ascontiguousarray(r, np.float32).reshape(-1, 5 + classes) for r in rows_per_image_list]
    counts = np.array([r.shape[0] for r in rows], np.int32)
    flat = np.ascontiguousarray(np.concatenate(rows, 0) if rows else np.zeros((0, 5 + classes), np.float32))
    t = np.ascontiguousarray(truth, np.float32).reshape(-1, 6)
    ap = np.zeros(classes, np.float64); m = C.c_double(0); st = np.zeros(8, np.float32)
    r = lib().yb_map_evaluate(flat.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), len(rows), classes,
                              t.ctypes.data_as(C.c_void_p), t.shape[0], iou_thresh, thresh_calc_avg_iou,
                              ap.ctypes.data_as(C.c_void_p), C.byref(m), st.ctypes.data_as(C.c_void_p))
    _check(r >= 0)
    keys = ("precision", "recall", "f1", "avg_iou", "tp", "fp", "fn", "detections")
    return float(m.value), ap, dict(zip(keys, (float(v) for v in st)))


def entropy_calibration(src: np.ndarray, bin_width: float = 1.0 / 16, max_bin: int = 4096) -> float:
    """``entropy_calibration`` of the reference (yolov2_forward_network_quantized.c:1292) on a host array."""
    a = np.ascontiguousarray(src, dtype=np.float32).ravel()
    r = float(lib().yb_entropy_calibration(a.ctypes.data_as(C.c_void_p), a.size, bin_width, max_bin))
    _check(r > 0)
    return r


def format_input_calibration(multipliers: np.ndarray) -> str:
    """The cfg line the reference writes to input_calibration.txt (yolov2_forward_network.c:753-769): per-convolution
    means over the calibration images printed with %g, closed by its constant 16."""
    m = np.asarray(multipliers, np.float32).reshape(-1, np.asarray(multipliers).shape[-1])
    mean = m.sum(axis=0, dtype=np.float32) / np.float32(m.shape[0])
    return "input_calibration = " + "".join("%g, " % v for v in mean) + "16"


# ---- the reference's function names -----------------------------------------------------------------------
def parse_network_cfg(filename: str, batch: int = 1, quantized: int = 0) -> Network:
    h = lib().yb_parse_network_cfg(filename.encode(), batch, quantized)
    _check(bool(h))
    return Network(h)


def load_weights_upto_cpu(net: Network, filename: str, cutoff: Optional[int] = None):
    _check(lib().yb_load_weights_upto(net._h, filename.encode(), net.n if cutoff is None else cutoff) == 0)


def yolov2_fuse_conv_batchnorm(net: Network):
    lib().yb_fuse_conv_batchnorm(net._h)


def calculate_binary_weights(net: Network):
    lib().yb_calculate_binary_weights(net._h)


def quantinization_and_get_multipliers(net: Network):
    lib().yb_quantinization_and_get_multipliers(net._h)


def network_predict_b200(net: Network, images: np.ndarray) -> np.ndarray:
    return net.predict(images, quantized=False)


def network_predict_b200_quantized(net: Network, images: np.ndarray) -> np.ndarray:
    return net.predict(images, quantized=True)


def network_predict_b200_cudnn_quantized(net: Network, images: np.ndarray) -> np.ndarray:
    """The reference's GPU INT8 mode (network_predict_gpu_cudnn_quantized): the INT8 layers are the parser's l.quantized."""
    return net.predict(images, quantized=YB_QUANT_GPU)


def load_network(cfg: str, weights: Optional[str], batch: int = 1, quantized: int = 0) -> Network:
    """The whole main.c:160-171 preparation sequence."""
    net = parse_network_cfg(cfg, batch, quantized)
    if weights:
        load_weights_upto_cpu(net, weights)
    yolov2_fuse_conv_batchnorm(net)
    calculate_binary_weights(net)
    if quantized:
        quantinization_and_get_multipliers(net)
    return net


def network_from_layers(descs: List[LayerDesc], batch: int, h: int, w: int, c: int, quantized: int = 0) -> Network:
    arr = (LayerDesc * len(descs))(*descs)
    hnd = lib().yb_network_from_layers(arr, len(descs), batch, h, w, c, quantized)
    _check(bool(hnd))
    return Network(hnd)


class PinnedBuffer:
    """cudaHostAlloc'ed buffer (float32 by default, or uint8 frames) for the end-to-end path."""

    def __init__(self, count: int, dtype=np.float32):
        self.count = count
        dt = np.dtype(dtype)
        self._p = lib().yb_alloc_pinned(count * dt.itemsize)
        if not self._p:
            raise YbError("cudaHostAlloc failed")
        ct = C.c_float if dt == np.float32 else C.c_uint8
        if dt not in (np.dtype(np.float32), np.dtype(np.uint8)):
            raise YbError("PinnedBuffer: float32 or uint8")
        self.array = np.ctypeslib.as_array(C.cast(self._p, C.POINTER(ct)), shape=(count,))

    def __del__(self):
        try:
            if self._p:
                lib().yb_free_pinned(self._p)
                self._p = None
        except Exception:
            pass
