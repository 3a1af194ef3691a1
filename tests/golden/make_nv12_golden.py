"""Writes tests/golden/nv12_cv2.npz: NV12 frames and OpenCV's cvtColor results for them, the yardstick of the NV12 device
frames (YB_FRAME_NV12).  Needs cv2; run from the repository root:

    python tests/golden/make_nv12_golden.py

Frames (key nv12_<i> [3h/2, w], rgb_<i> / bgr_<i> [h, w, 3] from COLOR_YUV2RGB_NV12 / COLOR_YUV2BGR_NV12):
  random frames of 2x2, 10x6, 64x48 and 4100x2 (wider than the resize kernel's shared-memory span of 4096 pixels);
  a 256x10 frame whose every row walks Y = 0..255, with (U, V) = (0, 0), (0, 255), (255, 0), (255, 255), (128, 128) on
  its five chroma rows.
"""
import os

import cv2
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "nv12_cv2.npz")


def frames():
    rng = np.random.default_rng(2024)
    out = [rng.integers(0, 256, size=(h * 3 // 2, w), dtype=np.uint8) for w, h in ((2, 2), (10, 6), (64, 48), (4100, 2))]
    walk = np.zeros((15, 256), np.uint8)
    walk[:10] = np.arange(256, dtype=np.uint8)
    for r, (u, v) in enumerate(((0, 0), (0, 255), (255, 0), (255, 255), (128, 128))):
        walk[10 + r, 0::2], walk[10 + r, 1::2] = u, v
    return out + [walk]


def main():
    data = {}
    for i, nv in enumerate(frames()):
        data[f"nv12_{i}"] = nv
        data[f"rgb_{i}"] = cv2.cvtColor(nv, cv2.COLOR_YUV2RGB_NV12)
        data[f"bgr_{i}"] = cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12)
    np.savez_compressed(OUT, **data)
    print(OUT, len(data) // 3, "frames, cv2", cv2.__version__)


if __name__ == "__main__":
    main()
