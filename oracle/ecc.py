"""NumPy restatement of the direct-method baseline: cv2.findTransformECC with MOTION_HOMOGRAPHY as
code/utils/direct_homography.py:8-57 calls it from code/homography_conventional_synthetic.py:186-223.

Chain: gray planes (augment, normalise, denorm_img, astype(uint8), cvtColor RGB2GRAY), 5x5 Gaussian, [-0.5, 0, 0.5]
gradients, warpPerspective with 1/32 px coordinates (INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0) and the
INTER_NEAREST mask, the ECC iterations, and the harness's post-processing.

`solve="fp64"` solves the 8x8 system in fp64 from fp64 sums, as libudh's kernel does; `solve="fp32"` mirrors cv2, which
stores the Hessian and the projections as float32 and inverts the Hessian with its own float32 LU.  Test-only: no GPU.
"""
import numpy as np

MEAN = (118.93, 113.97, 102.60)
STD = (69.85, 68.81, 72.45)
ECC_OK, ECC_NAN, ECC_NOCONV = 0, 1, 2
_INT_MIN, _INT_MAX = float(np.iinfo(np.int32).min), float(np.iinfo(np.int32).max)


# ---------------------------------------------------------------------------- input preparation
def augment_normalise(img_u8, five=None):
    """[H,W,3] uint8 -> the normalised fp32 image of the Dataloader: optional augmentation five = (gamma, brightness,
    colour R, G, B) with pow in fp64 rounded once to fp32, then (v - mean) / std in fp32 (I's statistics)."""
    v = img_u8.astype(np.float32)
    if five is not None:
        f = np.asarray(five, np.float32)
        v = np.power(v.astype(np.float64), np.float64(f[0])).astype(np.float32)
        v = v * f[1]
        v = v * f[2:5].reshape(1, 1, 3)
        v = np.clip(v, np.float32(0), np.float32(255))
    return (v - np.array(MEAN, np.float32)) / np.array(STD, np.float32)


def denorm_u8(img_norm):
    """utils.denorm_img(img).astype(np.uint8): float64 statistics, truncation."""
    d = img_norm * np.array(STD).reshape(1, 1, 3) + np.array(MEAN).reshape(1, 1, 3)
    return np.clip(np.trunc(d), 0, 255).astype(np.uint8)


def rgb2gray_u8(rgb):
    """cv2.cvtColor(rgb, COLOR_RGB2GRAY) on uint8: 15-bit fixed point, round half up."""
    c = rgb.astype(np.int64)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + 16384) >> 15).astype(np.uint8)


def prep(I_u8, Ip_u8, aug=None):
    """Batched: decoded I, I' [B,H,W,3] uint8 and the [B,11] augmentation table -> gray planes [B,H,W] uint8 x 2."""
    B = I_u8.shape[0]
    g1 = np.empty(I_u8.shape[:3], np.uint8); g2 = np.empty_like(g1)
    for b in range(B):
        on = aug is not None and float(aug[b][0]) != 0.0
        a1 = np.asarray(aug[b][1:6]) if on else None
        a2 = np.asarray(aug[b][6:11]) if on else None
        g1[b] = rgb2gray_u8(denorm_u8(augment_normalise(I_u8[b], a1)))
        g2[b] = rgb2gray_u8(denorm_u8(augment_normalise(Ip_u8[b], a2)))
    return g1, g2


# ---------------------------------------------------------------------------- pre-pass
def blur(u8):
    """GaussianBlur(float32(u8), (5,5), 0, 0): kernel [1,4,6,4,1]/16, BORDER_REFLECT_101.  Exact in fp32."""
    k = np.array([1, 4, 6, 4, 1], np.float32) / np.float32(16)
    p = np.pad(u8.astype(np.float32), 2, mode="reflect")
    H, W = u8.shape
    r = sum(k[j] * p[:, j:j + W] for j in range(5))
    return sum(k[i] * r[i:i + H, :] for i in range(5)).astype(np.float32)


def gradients(b):
    """filter2D(b, -1, [-0.5, 0, 0.5]) and its transpose, BORDER_REFLECT_101 (zero on the first / last column / row)."""
    gx = np.zeros_like(b); gy = np.zeros_like(b)
    gx[:, 1:-1] = np.float32(0.5) * (b[:, 2:] - b[:, :-2])
    gy[1:-1, :] = np.float32(0.5) * (b[2:, :] - b[:-2, :])
    return gx, gy


# ---------------------------------------------------------------------------- warp
def warp_map(W, H, Wd):
    """Per template pixel: top-left source pixel, the 1/32 px fractions and the INTER_NEAREST mask of src = W (x, y, 1)."""
    M = np.asarray(W, np.float32).astype(np.float64).reshape(9)
    ys, xs = np.mgrid[0:H, 0:Wd].astype(np.float64)
    X0 = M[0] * xs + M[1] * ys + M[2]
    Y0 = M[3] * xs + M[4] * ys + M[5]
    W0 = M[6] * xs + M[7] * ys + M[8]
    with np.errstate(divide="ignore", invalid="ignore"):
        wl = np.where(W0 != 0, 32.0 / W0, 0.0)
        wn = np.where(W0 != 0, 1.0 / W0, 0.0)
    q = lambda v: np.rint(np.clip(np.nan_to_num(v, nan=0.0), _INT_MIN, _INT_MAX)).astype(np.int64)
    X, Y = q(X0 * wl), q(Y0 * wl)
    Xn, Yn = q(X0 * wn), q(Y0 * wn)
    xi = np.clip(X >> 5, -32768, 32767); yi = np.clip(Y >> 5, -32768, 32767)
    ax = (X & 31).astype(np.float32) / np.float32(32); ay = (Y & 31).astype(np.float32) / np.float32(32)
    mask = (Xn >= 0) & (Xn < Wd) & (Yn >= 0) & (Yn < H)
    return xi, yi, ax, ay, mask


def bilinear(plane, xi, yi, ax, ay):
    H, Wd = plane.shape
    def at(y, x):
        ok = (x >= 0) & (x < Wd) & (y >= 0) & (y < H)
        return np.where(ok, plane[np.clip(y, 0, H - 1), np.clip(x, 0, Wd - 1)], np.float32(0)).astype(np.float32)
    one = np.float32(1)
    w00, w01, w10, w11 = (one - ay) * (one - ax), (one - ay) * ax, ay * (one - ax), ay * ax
    return ((at(yi, xi) * w00 + at(yi, xi + 1) * w01) + at(yi + 1, xi) * w10) + at(yi + 1, xi + 1) * w11


def warp_linear(plane, W):
    """cv2.warpPerspective(plane, W, size, INTER_LINEAR | WARP_INVERSE_MAP), BORDER_CONSTANT 0."""
    xi, yi, ax, ay, _ = warp_map(W, *plane.shape)
    return bilinear(plane, xi, yi, ax, ay)


# ---------------------------------------------------------------------------- iterations
def _lu_inv_f32(A):
    """cv2 Mat::inv (DECOMP_LU) on float32: Gaussian elimination with partial pivoting on [A | I], back substitution."""
    A = np.array(A, np.float32); n = A.shape[0]
    b = np.eye(n, dtype=np.float32)
    for i in range(n):
        k = i + int(np.argmax(np.abs(A[i:, i])))
        if abs(A[k, i]) < np.float32(np.finfo(np.float32).eps * 10):
            return np.zeros_like(A)
        if k != i:
            A[[i, k]] = A[[k, i]]; b[[i, k]] = b[[k, i]]
        d = np.float32(-1) / A[i, i]
        for j in range(i + 1, n):
            alpha = A[j, i] * d
            A[j, i + 1:] += alpha * A[i, i + 1:]
            b[j] += alpha * b[i]
        A[i, i] = -d
    for i in range(n - 1, -1, -1):
        for j in range(n):
            s = b[i, j]
            for k in range(i + 1, n):
                s = np.float32(s - A[i, k] * b[k, j])
            b[i, j] = s * A[i, i]
    return b


def ecc(template_u8, image_u8, W_init=None, max_iters=8, eps=1e-10, solve="fp64", trace=None):
    """-> dict(W [3,3] float32, rho, iters, status) for one pair.  `trace` (a list) receives per iteration the quantities
    that decide the outcome: rho and lambda_d, and the sums they come from (correlation, Hessian, projections)."""
    H, Wd = template_u8.shape
    T = blur(template_u8); Ib = blur(image_u8)
    gx, gy = gradients(Ib)
    W = np.eye(3, dtype=np.float32) if W_init is None else np.array(W_init, np.float32).reshape(3, 3).copy()
    ys, xs = np.mgrid[0:H, 0:Wd].astype(np.float32)
    rho, last, status, it = -1.0, -eps, ECC_OK, 0
    i = 1
    while i <= max_iters and abs(rho - last) >= eps:
        it = i
        xi, yi, ax, ay, mask = warp_map(W, H, Wd)
        Iw = bilinear(Ib, xi, yi, ax, ay)
        gxw = bilinear(gx, xi, yi, ax, ay); gyw = bilinear(gy, xi, yi, ax, ay)
        n = float(mask.sum())
        if n > 0:
            iw64, t64 = Iw[mask].astype(np.float64), T[mask].astype(np.float64)
            mI, mT = iw64.sum() / n, t64.sum() / n
            sdI = np.sqrt(max((iw64 * iw64).sum() / n - mI * mI, 0.0)); sdT = np.sqrt(max((t64 * t64).sum() / n - mT * mT, 0.0))
        else:
            mI = mT = sdI = sdT = 0.0
        imgNorm, tmpNorm = np.sqrt(n * sdI * sdI), np.sqrt(n * sdT * sdT)
        Iz = np.where(mask, Iw - np.float32(mI), Iw).astype(np.float32)
        Tz = np.where(mask, T - np.float32(mT), np.float32(0)).astype(np.float32)
        h = W.reshape(9)
        den = xs * h[6] + ys * h[7] + np.float32(1)
        hatX = (-xs * h[0] - ys * h[1] - h[2]) / den
        hatY = (-xs * h[3] - ys * h[4] - h[5]) / den
        gxd, gyd = gxw / den, gyw / den
        tmp = hatX * gxd + hatY * gyd
        J = np.stack([gxd * xs, gyd * xs, tmp * xs, gxd * ys, gyd * ys, tmp * ys, gxd, gyd]).reshape(8, -1).astype(np.float64)
        Hs = J @ J.T
        ip = J @ Iz.reshape(-1).astype(np.float64)
        tp = J @ Tz.reshape(-1).astype(np.float64)
        corr = float(Tz.reshape(-1).astype(np.float64) @ Iz.reshape(-1).astype(np.float64))
        with np.errstate(divide="ignore", invalid="ignore"):
            last, rho = rho, corr / (imgNorm * tmpNorm)
        if solve == "fp32":
            Hinv = _lu_inv_f32(Hs.astype(np.float32))
            ip32, tp32 = ip.astype(np.float32), tp.astype(np.float32)
            ipH = (Hinv.astype(np.float64) @ ip32.astype(np.float64)).astype(np.float32)
            lambda_n = imgNorm * imgNorm - float(ip32.astype(np.float64) @ ipH.astype(np.float64))
            lambda_d = corr - float(tp32.astype(np.float64) @ ipH.astype(np.float64))
        else:
            try:
                sol = np.linalg.solve(Hs, np.stack([ip, tp], 1))
            except np.linalg.LinAlgError:                       # the kernel's LU divides by the zero pivot: NaN from here on
                sol = np.full((8, 2), np.nan)
            lambda_n = imgNorm * imgNorm - float(ip @ sol[:, 0])
            lambda_d = corr - float(tp @ sol[:, 0])
        if trace is not None:
            trace.append(dict(rho=rho, lambda_d=lambda_d, corr=corr, hessian=Hs, ip=ip, tp=tp))
        if np.isnan(rho):
            status = ECC_NAN; break
        if lambda_d <= 0.0:
            status = ECC_NOCONV; break
        lam = lambda_n / lambda_d
        if solve == "fp32":
            err = (np.float32(lam) * Tz - Iz).astype(np.float32)
            ep = (J @ err.reshape(-1).astype(np.float64)).astype(np.float32)
            dp = (Hinv.astype(np.float64) @ ep.astype(np.float64)).astype(np.float32)
        else:
            dp = (lam * sol[:, 1] - sol[:, 0]).astype(np.float32)
        flat = W.reshape(9)
        for k, s in enumerate((0, 3, 6, 1, 4, 7, 2, 5)):     # update_warping_matrix_ECC
            flat[s] = np.float32(flat[s] + dp[k])
        W = flat.reshape(3, 3)
        i += 1
    return dict(W=W, rho=rho, iters=it, status=status)


# ---------------------------------------------------------------------------- post-processing
def h4p(W, status, pts1, gt=None, rho=45.0):
    """direct_homography.py:42-57 + homography_conventional_synthetic.py:204-223 for one sample:
    -> (pred_h4p [8] float32, h_loss or None, fail code or None) with fail 1 = not found, 2 = worse than identity."""
    pts = np.asarray(pts1, np.float32).reshape(4, 2)
    found = status == ECC_OK
    pred = np.zeros(8, np.float32)
    if found:
        try:
            Mi = np.linalg.inv(np.asarray(W, np.float32).astype(np.float64).reshape(3, 3))
        except np.linalg.LinAlgError:
            found = False
    if found:
        for k in range(4):
            x, y = float(pts[k, 0]), float(pts[k, 1])
            s = x * Mi[2, 0] + y * Mi[2, 1] + Mi[2, 2]
            X = Y = np.float32(0)
            if abs(s) > np.finfo(np.float32).eps:
                s = 1.0 / s
                X = np.float32((x * Mi[0, 0] + y * Mi[0, 1] + Mi[0, 2]) * s)
                Y = np.float32((x * Mi[1, 0] + y * Mi[1, 1] + Mi[1, 2]) * s)
            pred[2 * k] = X - pts[k, 0]; pred[2 * k + 1] = Y - pts[k, 1]
    pred[pred >= rho] = 2 * rho
    pred[pred <= -rho] = -2 * rho
    if gt is None:
        return pred, None, None
    g = np.asarray(gt, np.float64).reshape(8)
    hl = float(np.sqrt(np.mean((pred.astype(np.float64) - g) ** 2)))
    ident = float(np.sqrt(np.mean(g ** 2)))
    fail = 0
    if not found:
        fail = 1
    elif ident < hl:
        fail, hl = 2, ident
    return pred, hl, fail
