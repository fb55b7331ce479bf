"""GPU tests of the mosaic's multi-band blend: udh_mosaic_multiband_u8 against cv2.detail_MultiBandBlender (oracle/multiband.py)
byte for byte, order and run independence, every level's sums against the NumPy restatement, a synthetic sweep stitched
with its true homographies against the texture it was cut from, and mosaic_images.py --blend multiband end to end."""
import os
import sys

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _mosaic_sweep as SW  # noqa: E402
import test_gpu_mosaic as GM  # noqa: E402
from oracle import multiband as MB  # noqa: E402

pytestmark = pytest.mark.gpu


def _blend(frames, M, canvas, bands, levels=False):
    from unsuperviseddeephomographyral2018_b200 import ops
    r = ops.mosaic_multiband_u8([torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames], M, canvas[0], canvas[1], bands,
                                levels=levels)
    return tuple(x.cpu().numpy() if isinstance(x, torch.Tensor) else [t.cpu().numpy() for t in x] for x in r)


def overlap_case(n=130, seed=3):
    """n frames of 24 x 30 stacked within a few pixels of each other: more than 128 overlap, so the int16 sums wrap."""
    rng = np.random.default_rng(seed)
    frames = [rng.integers(0, 256, (24, 30, 3), np.uint8) for _ in range(n)]
    M = np.stack([GM.T(2 + (k % 5), 3 + (k % 3)) for k in range(n)])
    return frames, M, (33, 41)


@pytest.mark.parametrize("bands", [0, 1, 5, 8])
@pytest.mark.parametrize("name", ["one", "two", "seven"])
def test_kernel_equals_the_oracle(name, bands):
    frames, M, canvas = GM._case(name, 3, np.random.default_rng(bands))
    got, mask = _blend(frames, M, canvas, bands)
    ref, ref_mask = MB.blend(frames, M, canvas[0], canvas[1], bands)
    assert np.array_equal(mask, ref_mask) and np.array_equal(got, ref)
    assert 0 < (mask == 255).sum() < mask.size


def test_kernel_equals_the_oracle_on_camera_frames():
    """Three 3000 x 4000 frames of a sweep, about 60 % overlap between neighbours."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(3, 3000, 4000, seed=5)
    G, ref = mosaic.chain_to_reference(H)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, ref)
    assert kept.all()
    got, mask = _blend(frames, M, (Hc, Wc), 5)
    ref_img, ref_mask = MB.blend(frames, M, Hc, Wc, 5)
    assert np.array_equal(mask, ref_mask) and np.array_equal(got, ref_img)


def test_kernel_equals_the_oracle_where_the_sums_wrap():
    frames, M, canvas = overlap_case()
    got, mask = _blend(frames, M, canvas, 3)
    ref, ref_mask = MB.blend(frames, M, canvas[0], canvas[1], 3)
    assert np.array_equal(mask, ref_mask) and np.array_equal(got, ref)
    assert (mask == 0).any()                                     # the wrapped weight sum reads as <= 0 there


def test_order_and_run_independence():
    frames, M, canvas = GM._case("seven", 3, np.random.default_rng(7))
    a = _blend(frames, M, canvas, 5)
    b = _blend(frames, M, canvas, 5)
    perm = [4, 1, 6, 0, 3, 5, 2]
    c = _blend([frames[k] for k in perm], M[perm], canvas, 5)
    for x in (b, c):
        assert np.array_equal(a[0], x[0]) and np.array_equal(a[1], x[1])


@pytest.mark.parametrize("case", ["seven", "wrap"])
def test_every_level_equals_the_restatement(case):
    """The canvas pyramid's acc / wacc as the feeds leave it, level by level: a failure names the level."""
    if case == "wrap":
        frames, M, canvas, bands = overlap_case() + (3,)
    else:
        frames, M, canvas = GM._case("seven", 3, np.random.default_rng(11))
        bands = 5
    got, mask, pyr = _blend(frames, M, canvas, bands, levels=True)
    r = MB.restate(*MB.fed(frames, M, canvas[0], canvas[1]), canvas[0], canvas[1], bands)
    assert len(pyr) == r["bands"] + 1
    for i, lv in enumerate(pyr):
        assert np.array_equal(lv[..., :3], r["acc"][i]), "level %d: acc" % i
        assert np.array_equal(lv[..., 3], r["wacc"][i]), "level %d: wacc" % i
    assert np.array_equal(got, r["mosaic"]) and np.array_equal(mask, r["mask"])


def test_rejects_bad_arguments():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    f = torch.zeros(8, 8, 3, dtype=torch.uint8, device="cuda")
    g = torch.zeros(8, 8, 1, dtype=torch.uint8, device="cuda")
    I = np.eye(3)[None]
    for frames, M, dh, dw, bands in (([f], I, 8, 8, 11), ([f], I, 8, 8, -1), ([f], I, 32767, 8, 0), ([g], I, 8, 8, 0),
                                     ([f], np.stack([I[0]] * 2), 8, 8, 0), ([f.float()], I, 8, 8, 0)):
        with pytest.raises(_lib.UdhError):
            ops.mosaic_multiband_u8(frames, M, dh, dw, bands)
    behind = np.array([[1.0, 0, 0], [0, 1.0, 0], [-0.2, 0, 1.0]])[None]     # x = 5 maps with a denominator of 0
    for M in (behind, np.full((1, 3, 3), np.nan)):
        with pytest.raises(ValueError):
            ops.mosaic_multiband_u8([f], M, 8, 8, 2)


def test_true_homographies_rebuild_the_texture():
    """A sweep cut from one texture, chained with its true pair homographies and blended across 5 bands: the mosaic equals
    the oracle, and on covered pixels it is the texture as the reference frame sees it.  Measured on one H100 80 GB HBM3:
    MAD 5.34 levels (the feathered blend: 0.22).  Most of it is cv2's CV_16S rule itself: every level is normalised by
    wacc + 1 with a truncating division, so one frame blended alone differs from its own warp by 3.1 levels at 5 bands
    (1.0 at 0 bands).  The bound is the measured value plus about 10 %; shifting the two end frames by 2 px raises the
    MAD to 8.2 (oracle, same sweep)."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    n, h, w = 6, 240, 320
    tex, frames, A, H = SW.sweep(n, h, w, seed=2)
    G, r = mosaic.chain_to_reference(H)
    M, (Hc, Wc), kept = mosaic.canvas([(h, w)] * n, G, r)
    got, mask = _blend(frames, M, (Hc, Wc), 5)
    ref_img, ref_mask = MB.blend(frames, M, Hc, Wc, 5)
    assert np.array_equal(got, ref_img) and np.array_equal(mask, ref_mask)
    seen = cv2.warpPerspective(tex, A[r] @ np.linalg.inv(M[r]), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    cov = mask == 255
    mad = np.abs(got.astype(np.int32) - seen.astype(np.int32))[cov].mean()
    print("canvas %dx%d, %.1f %% covered, MAD %.3f" % (Hc, Wc, 100 * cov.mean(), mad))
    assert cov.mean() > 0.7 and mad <= 5.9


def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import ops
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(4, 240, 320, seed=9)
    names = ["DSC_%04d.JPG" % k for k in range(4)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband"]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[0] == "canvas" and head[3] == "ref" and head[5:] == ["blend", "multiband", "5"]
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms = [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        assert parts[0] == nm and parts[1] in ("kept", "dropped")
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm)))
            Ms.append(np.array([float(v) for v in parts[2:]]).astype(np.float32).astype(np.float64).reshape(3, 3))
    mos, _ = MB.blend(imgs, np.stack(Ms), Hc, Wc, 5)                  # BGR in, BGR out: the blender treats channels alike
    assert (out / "mosaic.jpg").read_bytes() == ops.encode_jpeg(mos[None])[0]
