"""Writes tests/golden/gen_golden.npz: the reference's own numpy_transformer (code/utils/numpy_spatial_transformer.py,
imported with its plotting imports stubbed) on the generator's geometry, the way gen_synthetic_data.py:63-64 calls it.

Two 240x320 BGR images (smooth textures, so the file stays small), each with one pair drawn as the generator draws
it (rho 45, patch 128: the warped images include out-of-image pixels).  Colour is warped one channel at a time (the
reference's 3-D branch relies on an old-NumPy expand_dims leniency); the gray image is cv2.cvtColor(bgr, COLOR_RGB2GRAY).
Stored: bgr, H_inverse, gray, warped (colour) and warped_gray.  Only data goes into the repository.

    python tests/golden/make_gen_golden.py [/path/to/reference/code]
"""
import os
import random
import sys
import types

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(ROOT), "reference", "code")
sys.path.insert(0, ROOT)

from unsuperviseddeephomographyral2018_b200 import gen_data as G     # noqa: E402


def load_reference_numpy_transformer():
    for name in ("matplotlib", "matplotlib.pyplot", "skimage", "skimage.io"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["skimage"].io = sys.modules["skimage.io"]
    sys.path.insert(0, os.path.join(REF, "utils"))
    import numpy_spatial_transformer as nst
    return nst


def main():
    nst = load_reference_numpy_transformer()
    rnd = random.Random(11)
    h, w = 240, 320
    bgr, hinv, gray, warped, warped_gray = [], [], [], [], []
    for k in range(2):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.stack([128 + 90 * np.sin(xx / (9.0 + 3 * c + k)) * np.cos(yy / (13.0 + 2 * c)) for c in range(3)], -1)
        img = (np.clip(img, 0, 255).astype(np.uint8) // 4) * 4       # smooth and coarse: the file stays small
        g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
        four, pert = G.pair_draws(rnd, 45, 128, h, w)
        H = cv2.getPerspectiveTransform(np.float32(four), np.float32(pert))
        Hi = np.linalg.inv(H)
        warped.append(np.stack([nst.numpy_transformer(img[..., c], Hi, (w, h)) for c in range(3)], axis=2))
        warped_gray.append(nst.numpy_transformer(g, Hi, (w, h)))
        bgr.append(img); hinv.append(Hi); gray.append(g)
    out = os.path.join(ROOT, "tests", "golden", "gen_golden.npz")
    np.savez_compressed(out, bgr=np.stack(bgr), H_inverse=np.stack(hinv), gray=np.stack(gray), warped=np.stack(warped),
                        warped_gray=np.stack(warped_gray))
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


if __name__ == "__main__":
    main()
