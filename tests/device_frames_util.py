"""Helpers of the device-frame tests: the NV12 -> RGB conversion restated in numpy, and device frames laid out in memory
the way decoders and strided views lay them out (padded pitch, odd start address, a frame that ends on the last byte of
its allocation)."""
import os

import numpy as np

GOLDEN_NV12 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nv12_cv2.npz")

# BT.601 limited range, OpenCV's fixed-point constants (cvtColor COLOR_YUV2RGB_NV12), 20 fractional bits
CY, CVR, CVG, CUG, CUB, SHIFT = 1220542, 1673527, -852492, -409993, 2116026, 20


def nv12_to_rgb(nv12):
    """uint8 NV12 [3h/2, w] (Y rows, then h/2 rows of interleaved U, V) -> uint8 RGB [h, w, 3]."""
    nv12 = np.asarray(nv12, np.uint8)
    h, w = nv12.shape[0] // 3 * 2, nv12.shape[1]
    Y = nv12[:h].astype(np.int64)
    uv = nv12[h:].reshape(h // 2, w // 2, 2).astype(np.int64)
    U = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1) - 128
    V = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1) - 128
    yy = np.maximum(0, Y - 16) * CY + (1 << (SHIFT - 1))
    r = (yy + CVR * V) >> SHIFT
    g = (yy + CVG * V + CUG * U) >> SHIFT
    b = (yy + CUB * U) >> SHIFT
    return np.stack([r, g, b], -1).clip(0, 255).astype(np.uint8)


def equivalent_host_frame(fmt, frame):
    """The packed RGB host frame a device frame stands for.  frame: rgb / bgr [h, w, 3], planar [3, h, w], nv12 [3h/2, w]."""
    if fmt == "rgb":
        return np.ascontiguousarray(frame)
    if fmt == "bgr":
        return np.ascontiguousarray(frame[..., ::-1])
    if fmt == "planar":
        return np.ascontiguousarray(frame.transpose(1, 2, 0))
    return nv12_to_rgb(frame)


def random_frame(fmt, w, h, rng):
    """A random frame of format fmt and size w x h, in the shape equivalent_host_frame takes."""
    shape = {"rgb": (h, w, 3), "bgr": (h, w, 3), "planar": (3, h, w), "nv12": (h * 3 // 2, w)}[fmt]
    return rng.integers(0, 256, size=shape, dtype=np.uint8)


# memory layouts of a device frame: (row padding in bytes, start offset in the allocation)
LAYOUTS = {"padded": (13, 0), "odd_offset": (5, 1), "tight": (0, 0)}


def device_frame(fmt, frame, layout, device="cuda", nv12_pair=False):
    """frame (as random_frame makes it) -> a torch uint8 view on the device in the given layout; the padding bytes are 0xAB.
    The tensor's storage holds exactly the bytes the view addresses from its start offset on, so the frame's last byte is
    the storage's last byte.  nv12_pair: (Y, UV) views of two storages with the same pitch."""
    import torch
    pad, off = LAYOUTS[layout]
    if fmt == "nv12" and nv12_pair:
        h = frame.shape[0] // 3 * 2
        return device_frame("plane", frame[:h], layout, device), device_frame("plane", frame[h:], layout, device)
    if fmt in ("rgb", "bgr"):
        h, w, _ = frame.shape
        pitch = 3 * w + pad
        shape, strides, size = (h, w, 3), (pitch, 3, 1), (h - 1) * pitch + 3 * w
    elif fmt == "planar":
        _, h, w = frame.shape
        pitch = w + pad
        plane = pitch * h + pad
        shape, strides, size = (3, h, w), (plane, pitch, 1), 2 * plane + (h - 1) * pitch + w
    else:   # nv12 [3h/2, w] or one plane [rows, w]
        rows, w = frame.shape
        pitch = w + pad
        shape, strides, size = (rows, w), (pitch, 1), (rows - 1) * pitch + w
    buf = np.full(off + size, 0xAB, np.uint8)
    np.lib.stride_tricks.as_strided(buf[off:], shape=shape, strides=strides)[...] = frame
    dev = torch.from_numpy(buf).to(device)
    return torch.as_strided(dev, shape, strides, off)
