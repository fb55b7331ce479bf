"""Host logic of report.py (CPU): the integer conversions of the points (checked against the cv2 call sequence from
float points in tests/test_draw_oracle.py test_composition), the file names and the global image index."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from unsuperviseddeephomographyral2018_b200 import report  # noqa: E402


def test_conversions():
    v = report.report_vertices(np.float32([[1.9, -1.9]] * 4), np.float32([[2.5, 3.5]] * 4), np.float32([[np.nan, 7.9]] * 4), 320)
    assert v[0].tolist() == [-2 ** 31, 7]                             # np.int32(nan) = INT_MIN, truncation
    assert v[4].tolist() == [322, 3]                                  # kp2 truncated after the offset
    assert v[8].tolist() == [1, -1] and v[12].tolist() == [1, -1]    # kp1 truncated toward zero
    assert v[16].tolist() == [322, 4]                                 # end2 = np.round(corr2): half to even


def test_synthetic_name_and_points():
    assert report.synthetic_name(3, 4, "l1_loss", 12.345678901) == "12_l1_loss_loss_" + str(np.float32(12.345678901)) + ".jpg"
    c1, c2, pr = report.synthetic_points(np.arange(8), np.ones(8), -np.ones(8))
    assert c1.dtype == np.float32 and c1.shape == (1, 4, 2)
    assert (c2 - c1 == 1).all() and (pr - c1 == -1).all()


def test_real_names_and_global_index():
    assert report.real_cnn_name(37, 1.25) == "37_Unsupervised__loss_1.25.jpg"
    assert report.conventional_name(5, 0.5) == "5_loss_0.5.jpg"
    # one rank: the reference's step*batch_size + i
    assert [report.global_index(0, 4, 2, 4, i) for i in range(4)] == [8, 9, 10, 11]
    # two ranks of 2 samples each on a global batch of 4: every index of the step once, rank 0 first
    ks = sorted(report.global_index(r, 2, 3, 4, i) for r in range(2) for i in range(2))
    assert ks == [12, 13, 14, 15]
    assert report.global_index(1, 2, 3, 4, 0) == 14


def test_clicked_points():
    g = np.arange(32, dtype=np.float32).reshape(2, 16) + 0.5
    c1, c2 = report.clicked_points(g)
    assert c1.dtype == np.float32 and c1.shape == (2, 4, 2)
    np.testing.assert_array_equal(c1[1].ravel(), g[1, :8] / 2)
    np.testing.assert_array_equal(c2[0].ravel(), g[0, 8:] / 2)
