"""Regenerate ecc_golden.npz: OpenCV's findTransformECC (MOTION_HOMOGRAPHY, 8 iterations, eps 1e-10, as
code/homography_conventional_synthetic.py runs it) on the gray planes of oracle.make_batch(seed=3, B=12), sample 0 with
photometric augmentation.  Needs cv2; the inputs are regenerated from the seed, only cv2's outputs are stored.

    python tests/golden/make_ecc_golden.py
"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ecc as E  # noqa: E402
from oracle import oracle as O  # noqa: E402

AUG0 = [1, 1.1, 1.3, 0.9, 1.05, 1.15, 0.85, 0.7, 1.1, 0.95, 1.0]


def main():
    import cv2
    b = O.make_batch(3, 12)
    aug = np.zeros((12, 11), np.float32); aug[0] = AUG0
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    K = 8
    W = np.zeros((12, 9), np.float32); rho = np.full(12, np.nan); status = np.zeros(12, np.int32)
    for s in range(12):
        try:
            r, w = cv2.findTransformECC(g1[s], g2[s], np.eye(3, dtype=np.float32), cv2.MOTION_HOMOGRAPHY,
                                        (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, K, 1e-10), None, 5)
            W[s], rho[s] = w.reshape(9), r
        except cv2.error as e:
            status[s] = E.ECC_NAN if "NaN" in str(e) else E.ECC_NOCONV
    np.savez_compressed(os.path.join(HERE, "ecc_golden.npz"), crc_gray_I=np.uint32(zlib.crc32(g1.tobytes())), crc_gray_I_prime=np.uint32(zlib.crc32(g2.tobytes())), W=W, rho=rho, status=status,
                        max_iters=np.int32(K), cv2_version=np.array(cv2.__version__))
    print("status", status.tolist())


if __name__ == "__main__":
    main()
