"""GPU tests of the sequence mosaic: udh_mosaic_blend_u8 against its restatement oracle/mosaic.py byte for byte, order and
run independence, a synthetic sweep mosaicked with its true homographies against the texture it was cut from, and
mosaic_images.py end to end."""
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
from oracle import mosaic as OM  # noqa: E402

pytestmark = pytest.mark.gpu


def T(dx, dy):
    return np.array([[1.0, 0, dx], [0, 1.0, dy], [0, 0, 1.0]])


def _case(name, C, rng):
    """(frames uint8 [h,w,C], M [n,3,3], canvas (Hc, Wc)) of a named case."""
    c, s = np.cos(0.4), np.sin(0.4)
    rot = T(60, 20) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    persp = np.array([[0.9, 0.05, 80.0], [-0.03, 1.05, -10.0], [4e-4, -2e-4, 1.0]])
    if name == "one":                                   # partly outside a canvas whose width is not a multiple of 64
        sizes, M, canvas = [(37, 53)], [T(-11.5, 9.25)], (41, 77)
    elif name == "two":                                 # mixed sizes, a canvas under 16 rows
        sizes, M, canvas = [(37, 53), (20, 30)], [T(-3, -20), persp @ T(-70, 0)], (13, 150)
    elif name == "seven":                               # x8 and x1/8 frames, a singular M, rotation, perspective, 1080x1920
        sizes = [(37, 53), (1080, 1920), (9, 11), (480, 640), (60, 80), (30, 30), (240, 320)]
        M = [T(5.5, 3.25), T(300, 40) @ np.diag([0.5, 0.5, 1.0]), T(900, 200) @ np.diag([8.0, 8.0, 1.0]),
             T(1000.25, 500.5) @ np.diag([0.125, 0.125, 1.0]), rot, np.array([[1.0, 2, 3], [2, 4, 6], [0, 0, 1]]), persp]
        canvas = (611, 1299)
    M = np.stack(M)
    frames = [rng.integers(0, 256, (h, w, C), np.uint8) for h, w in sizes]
    if name == "seven":
        frames[1] = SW.texture(rng, 1080, 1920)[..., :C].copy()
    return frames, M, canvas


def _blend(frames, M, canvas, feather):
    from unsuperviseddeephomographyral2018_b200 import ops
    out, mask = ops.mosaic_blend_u8([torch.from_numpy(f).cuda() for f in frames], M, canvas[0], canvas[1], feather)
    return out.cpu().numpy(), mask.cpu().numpy()


@pytest.mark.parametrize("feather", [0, 1, 64, 1024])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", ["one", "two", "seven"])
def test_kernel_equals_the_oracle(name, C, feather):
    frames, M, canvas = _case(name, C, np.random.default_rng(C * 10 + feather))
    got, mask = _blend(frames, M, canvas, feather)
    ref, ref_mask = OM.blend(frames, M, canvas[0], canvas[1], feather)
    assert np.array_equal(mask, ref_mask) and np.array_equal(got, ref)
    assert 0 < (mask == 255).sum() < mask.size


def test_kernel_equals_the_oracle_on_camera_frames():
    """Three 3000 x 4000 frames of a sweep, about 60 % overlap between neighbours."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(3, 3000, 4000, seed=5)
    G, ref = mosaic.chain_to_reference(H)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, ref)
    assert kept.all()
    got, mask = _blend(frames, M, (Hc, Wc), 64)
    ref_img, ref_mask = OM.blend(frames, M, Hc, Wc, 64)
    assert np.array_equal(mask, ref_mask) and np.array_equal(got, ref_img)


def test_order_and_run_independence():
    frames, M, canvas = _case("seven", 3, np.random.default_rng(7))
    a = _blend(frames, M, canvas, 64)
    b = _blend(frames, M, canvas, 64)
    perm = [4, 1, 6, 0, 3, 5, 2]
    c = _blend([frames[k] for k in perm], M[perm], canvas, 64)
    for x in (b, c):
        assert np.array_equal(a[0], x[0]) and np.array_equal(a[1], x[1])


def test_rejects_bad_arguments():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    f = torch.zeros(8, 8, 3, dtype=torch.uint8, device="cuda")
    g = torch.zeros(8, 8, 1, dtype=torch.uint8, device="cuda")
    I = np.eye(3)[None]
    for frames, M, dh, dw, feather in (([f], I, 8, 8, 1025), ([f], I, 8, 8, -1), ([f], I, 32767, 8, 0), ([f, g], np.stack([I[0]] * 2), 8, 8, 0),
                                       ([f], np.stack([I[0]] * 2), 8, 8, 0), ([f.float()], I, 8, 8, 0)):
        with pytest.raises(_lib.UdhError):
            ops.mosaic_blend_u8(frames, M, dh, dw, feather)


def test_true_homographies_rebuild_the_texture():
    """A sweep cut from one texture, chained with its true pair homographies: the mosaic equals the oracle, and on covered
    pixels it is the texture as the reference frame sees it (mean absolute difference <= 2 levels).  An inverted chain or a
    wrong canvas offset moves whole frames and fails the second check."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    n, h, w = 6, 240, 320
    tex, frames, A, H = SW.sweep(n, h, w, seed=2)
    for ref in (None, 0):
        G, r = mosaic.chain_to_reference(H, ref)
        M, (Hc, Wc), kept = mosaic.canvas([(h, w)] * n, G, r)
        assert kept.all() and Wc > 2.5 * w
        got, mask = _blend(frames, M, (Hc, Wc), 64)
        ref_img, ref_mask = OM.blend(frames, M, Hc, Wc, 64)
        assert np.array_equal(got, ref_img) and np.array_equal(mask, ref_mask)
        # canvas pixel -> reference frame (inv(T) = G_r inv(M_r)) -> texture (A_r)
        seen = cv2.warpPerspective(tex, A[r] @ np.linalg.inv(M[r]), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
        cov = mask == 255
        mad = np.abs(got.astype(np.int32) - seen.astype(np.int32))[cov].mean()
        print("ref %s: canvas %dx%d, %.1f %% covered, MAD %.3f" % (r, Hc, Wc, 100 * cov.mean(), mad))
        assert cov.mean() > 0.7 and mad <= 2.0


def test_cli_end_to_end(tmp_path):
    import align_images
    import mosaic_images as cli
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(4, 240, 320, seed=9)
    names = ["DSC_%04d.JPG" % k for k in range(4)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none")]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[0] == "canvas" and head[3] == "ref" and int(head[4]) == 2
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms = [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        assert parts[0] == nm and parts[1] in ("kept", "dropped")
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm)))
            Ms.append(np.array([float(v) for v in parts[2:]]).astype(np.float32).astype(np.float64).reshape(3, 3))
    mos, _ = OM.blend(imgs, np.stack(Ms), Hc, Wc, 64)
    ok, ref = cv2.imencode(".jpg", mos, [cv2.IMWRITE_JPEG_QUALITY, 95])
    assert (out / "mosaic.jpg").read_bytes() == ref.tobytes()
    (raw / "pairs.txt").write_text("".join("%s %s\n" % (names[k], names[k + 1]) for k in range(3)))
    al = tmp_path / "aligned"
    assert align_images.main(["--pairs", str(raw / "pairs.txt"), "--out_dir", str(al), "--save_warped", "False", "--seeded_weights",
                              "True", "--model_dir", str(tmp_path / "none")]) == 0
    assert (out / "pairs.txt").read_text() == (al / "homographies.txt").read_text()
