"""Generates tests/golden/canny_cv2.npz: OpenCV's cv2.Canny on a few small images, so the numpy statement of Canny in
tests/control_ref.py stays pinned on a machine without cv2.

Case i holds case{i}_img (uint8 (H, W, 3) or (H, W)), case{i}_thr ((low, high)) and case{i}_edges, cv2.Canny(img, low,
high) with the default 3 x 3 aperture and the L1 gradient.  Run from the repo root with OpenCV installed:
  python tests/golden/make_canny_golden.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))


def cases():
    from tests.control_ref import spiral

    rng = np.random.default_rng(19)
    noise = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
    blurred = cv2.GaussianBlur(rng.integers(0, 256, (64, 48, 3), dtype=np.uint8), (0, 0), 1.0)
    grey = cv2.GaussianBlur(rng.integers(0, 256, (33, 71), dtype=np.uint8), (0, 0), 1.5)
    flat = np.full((16, 24, 3), 77, dtype=np.uint8)
    return [(noise, (50, 200)), (blurred, (50, 200)), (grey, (50, 200)), (spiral(96, 96), (50, 200)),
            (blurred, (20, 90)), (flat, (50, 200))]


def main():
    out = {}
    for i, (img, (low, high)) in enumerate(cases()):
        out[f"case{i}_img"] = img
        out[f"case{i}_thr"] = np.array([low, high], dtype=np.int32)
        out[f"case{i}_edges"] = cv2.Canny(img, low, high)
    out["opencv_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "canny_cv2.npz"), **out)
    print(f"wrote {len(out) // 3} cases (OpenCV {cv2.__version__})")


if __name__ == "__main__":
    main()
