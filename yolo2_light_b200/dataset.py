"""Host-side dataset plumbing for the mAP tool (SURVEY 8f row 4): what ``validate_detector_map`` reads from disk
(additionally.c:4541-4600, 4662-4678) -- the ``data`` cfg (``valid = <list file>``, ``names = <file>``), the image list,
and per image a label file found by the reference's path rewriting (``images`` -> ``labels``, extension -> ``.txt``) with
lines ``class x y w h``.  Image decoding: uncompressed 24-bit BMP and binary PPM only (the reference uses stb_image;
no codec is vendored here)."""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import numpy as np


def read_data_cfg(path: str) -> Dict[str, str]:
    """``read_data_cfg`` (additionally.c:3301): ``key = value`` lines, ``#``/``;`` comments."""
    out: Dict[str, str] = {}
    for line in open(path):
        line = line.strip()
        if not line or line[0] in "#;" or "=" not in line:
            continue
        k, v = line.split("=", 1)
        out[k.strip()] = v.strip()
    return out


def label_path(image_path: str) -> str:
    """The reference's find_replace chain (additionally.c:4664-4670)."""
    p = image_path.replace("images", "labels", 1).replace("JPEGImages", "labels", 1)
    for ext in (".jpg", ".png", ".bmp", ".JPG", ".JPEG", ".ppm"):
        p = p.replace(ext, ".txt", 1)
    return p


def read_labels(path: str) -> np.ndarray:
    """``read_boxes`` (additionally.c:4441): float32 [n, 5] = class, x, y, w, h; a missing file is an empty set."""
    rows: List[Tuple[float, ...]] = []
    if os.path.exists(path):
        toks = open(path).read().split()
        for k in range(0, len(toks) - 4, 5):
            try:
                rows.append((float(int(toks[k])), *(float(t) for t in toks[k + 1:k + 5])))
            except ValueError:
                break                      # fscanf stops at the first malformed record
    return np.array(rows, np.float32).reshape(-1, 5)


def read_image_u8(path: str) -> np.ndarray:
    """uint8 [h, w, 3] RGB from a 24-bit uncompressed BMP or a binary PPM (P6, maxval 255)."""
    data = open(path, "rb").read()
    if data[:2] == b"BM":
        off = int.from_bytes(data[10:14], "little")
        w = int.from_bytes(data[18:22], "little", signed=True)
        h = int.from_bytes(data[22:26], "little", signed=True)
        bpp = int.from_bytes(data[28:30], "little")
        comp = int.from_bytes(data[30:34], "little")
        if bpp != 24 or comp != 0:
            raise ValueError(f"{path}: only uncompressed 24-bit BMP is supported")
        flip = h > 0
        h = abs(h)
        row = (3 * w + 3) // 4 * 4
        a = np.frombuffer(data, np.uint8, count=row * h, offset=off).reshape(h, row)[:, :3 * w].reshape(h, w, 3)
        a = a[:, :, ::-1]                  # BGR -> RGB
        return np.ascontiguousarray(a[::-1] if flip else a)
    if data[:2] == b"P6":
        toks: List[bytes] = []
        i = 2
        while len(toks) < 3:               # width, height, maxval, skipping whitespace and comments
            while data[i:i + 1].isspace():
                i += 1
            if data[i:i + 1] == b"#":
                while data[i:i + 1] != b"\n":
                    i += 1
                continue
            j = i
            while not data[j:j + 1].isspace():
                j += 1
            toks.append(data[i:j]); i = j
        w, h, mx = (int(t) for t in toks)
        if mx != 255:
            raise ValueError(f"{path}: only maxval 255 PPM is supported")
        return np.frombuffer(data, np.uint8, count=w * h * 3, offset=i + 1).reshape(h, w, 3).copy()
    raise ValueError(f"{path}: not a BMP / PPM file")


def load_validation_set(datacfg: str):
    """Returns (image paths, class names, truth float32 [n, 6] = image index, class, x, y, w, h)."""
    opt = read_data_cfg(datacfg)
    paths = [p.strip() for p in open(opt.get("valid", "data/train.txt")) if p.strip()]
    names = [n.strip() for n in open(opt["names"])] if "names" in opt and os.path.exists(opt["names"]) else []
    truth = []
    for k, p in enumerate(paths):
        for row in read_labels(label_path(p)):
            truth.append((float(k), *row))
    return paths, names, np.array(truth, np.float32).reshape(-1, 6)


def evaluate_map(net, paths, truth: np.ndarray, classes: int, iou_thresh: float = 0.5, thresh_calc_avg_iou: float = 0.24,
                 max_rows: int = 8192, quantized: bool = False, progress=None, mixed_sizes: bool = False):
    """The loop of ``validate_detector_map`` (additionally.c:4614-4780) around any object with ``batch``,
    ``predict_image_u8(images_u8[batch, h, w, 3], quantized=)`` and ``detect(w, h, thresh, nms, relative=, letter=,
    max_rows=, quantized=)`` -- ``yolo2_light_b200.Network`` -- then ``yb_map_evaluate``.  Returns (mAP, ap[classes], stats).

    mixed_sizes=True uses ``predict_frames_u8(list of [h_i, w_i, 3] frames, quantized=)`` and ``detect_frames(sizes, ...)``
    instead: every batch takes the next ``batch`` images whatever their sizes, and the last one is a partial batch, so a
    dataset whose images rarely share a size runs ``batch`` images per forward rather than about one."""
    from . import api
    rows = []
    B = net.batch
    done = 0

    def flush(chunk):
        nonlocal done
        n = len(chunk)
        while len(chunk) < B:
            chunk.append(chunk[-1])                                # pad the batch; its extra rows are dropped
        net.predict_image_u8(np.stack(chunk), quantized=quantized)
        # the reference's settings: thresh .005, nms .45, relative coordinates (get_network_boxes(net, 1, 1, ...), :4657)
        dets, counts = net.detect(1, 1, 0.005, 0.45, relative=0, letter=0, max_rows=max_rows, quantized=quantized)
        if max(counts[:n]) > max_rows:
            raise ValueError(f"{max(counts[:n])} candidates in one image, only {max_rows} kept: raise max_rows")
        rows.extend(dets[:n])
        done += n
        if progress:
            progress(done, len(paths))

    def flush_mixed(chunk):
        nonlocal done
        net.predict_frames_u8(chunk, quantized=quantized)
        dets, counts = net.detect_frames([(1, 1)] * len(chunk), 0.005, 0.45, relative=0, letter=0, max_rows=max_rows,
                                         quantized=quantized)
        if max(counts) > max_rows:
            raise ValueError(f"{max(counts)} candidates in one image, only {max_rows} kept: raise max_rows")
        rows.extend(dets)
        done += len(chunk)
        if progress:
            progress(done, len(paths))

    if mixed_sizes:
        for first in range(0, len(paths), B):
            flush_mixed([read_image_u8(p) for p in paths[first:first + B]])
        return api.map_evaluate(rows, truth, classes, iou_thresh, thresh_calc_avg_iou)
    chunk = []
    for p in paths:                                                # images of one size share a batch, order is kept
        img = read_image_u8(p)
        if chunk and (img.shape != chunk[0].shape or len(chunk) == B):
            flush(chunk)
            chunk = []
        chunk.append(img)
    if chunk:
        flush(chunk)
    return api.map_evaluate(rows, truth, classes, iou_thresh, thresh_calc_avg_iou)
