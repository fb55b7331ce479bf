"""NumPy restatement of the baseline-JPEG decoder of csrc/jpeg.cu (test infrastructure only, like oracle/ecc.py).

Decodes what the device decoder accepts (baseline Huffman, 8-bit, gray or YCbCr 4:4:4 / 4:2:2 / 4:2:0, restart
intervals) the way libjpeg-turbo does by default, i.e. what cv2.imread(..., IMREAD_COLOR)[..., ::-1] returns:
ISLOW integer IDCT (CONST_BITS 13, PASS1_BITS 2, output through the 10-bit wrapping range-limit table), fancy
upsampling (triangle filters, edge samples replicated; plain replication when the chroma plane is <= 2 samples wide)
and jdcolor's 16-bit fixed-point YCbCr -> RGB.  The Huffman decode is a plain per-symbol loop: slow, but only tests run it.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63])


class Unsupported(ValueError):
    pass


def _u16(d, i):
    return (d[i] << 8) | d[i + 1]


def parse(data):
    """Markers -> dict(h, w, comps=[(id, hs, vs, tq)], qt, dc, ac, scan=[(comp index, td, ta)], ri, entropy bytes)."""
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Unsupported("not a JPEG")
    i, qt, dc, ac, ri, frame = 2, {}, {}, {}, 0, None
    while True:
        while i < len(d) and d[i] == 0xFF and i + 1 < len(d) and d[i + 1] == 0xFF:
            i += 1
        if i + 4 > len(d) or d[i] != 0xFF:
            raise Unsupported("truncated header")
        m, ln = d[i + 1], _u16(d, i + 2)
        seg = d[i + 4:i + 2 + ln]
        if len(seg) != ln - 2:
            raise Unsupported("truncated header")
        if m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise Unsupported("not 8-bit")
            h, w, nc = _u16(seg, 1), _u16(seg, 3), seg[5]
            comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nc)]
            frame = (h, w, comps)
        elif m in (0xC2, 0xC3) or 0xC5 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported("not baseline")
        elif m == 0xDB:
            j = 0
            while j < len(seg):
                if seg[j] >> 4:
                    raise Unsupported("16-bit quantisation table")
                qt[seg[j] & 15] = np.array(list(seg[j + 1:j + 65]), np.int64)[np.argsort(ZIGZAG)]   # natural order
                j += 65
        elif m == 0xC4:
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                counts = list(seg[j + 1:j + 17])
                vals = list(seg[j + 17:j + 17 + sum(counts)])
                codes, code, k = {}, 0, 0
                for ln_ in range(1, 17):
                    for _ in range(counts[ln_ - 1]):
                        codes[(ln_, code)] = vals[k]; k += 1; code += 1
                    code <<= 1
                (ac if tc else dc)[th] = codes
                j += 17 + sum(counts)
        elif m == 0xDD:
            ri = _u16(seg, 0)
        elif m == 0xDA:
            if frame is None:
                raise Unsupported("no frame header")
            ids = [c[0] for c in frame[2]]
            scan = [(ids.index(seg[1 + 2 * k]), seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(seg[0])]
            return dict(h=frame[0], w=frame[1], comps=frame[2], qt=qt, dc=dc, ac=ac, scan=scan, ri=ri, entropy=d[i + 2 + ln:])
        i += 2 + ln


def _segments(ent):
    """Entropy-coded bytes -> list of bit lists, split at RSTn; FF00 unstuffed; stops at any other marker."""
    segs, cur, j = [], bytearray(), 0
    while j < len(ent):
        b = ent[j]
        if b == 0xFF and j + 1 < len(ent):
            nb = ent[j + 1]
            if nb == 0x00:
                cur.append(0xFF); j += 2; continue
            if 0xD0 <= nb <= 0xD7:
                segs.append(cur); cur = bytearray(); j += 2; continue
            if nb == 0xFF:
                j += 1; continue
            break
        cur.append(b); j += 1
    segs.append(cur)
    return segs


class _Bits:
    def __init__(self, buf):
        self.bits = np.unpackbits(np.frombuffer(bytes(buf), np.uint8)) if len(buf) else np.zeros(0, np.uint8)
        self.pos = 0

    def get(self, n):
        if self.pos + n > len(self.bits):
            raise EOFError("entropy data exhausted")
        v = 0
        for b in self.bits[self.pos:self.pos + n]:
            v = (v << 1) | int(b)
        self.pos += n
        return v

    def huff(self, codes):
        code = 0
        for ln in range(1, 17):
            code = (code << 1) | self.get(1)
            if (ln, code) in codes:
                return codes[(ln, code)]
        raise ValueError("invalid Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(p):
    """Quantised coefficients per component, [blocks_h, blocks_w, 64] in natural order."""
    comps, scan = p["comps"], p["scan"]
    if len(comps) == 1:
        hs = vs = [1]; hmax = vmax = 1
    else:
        hs, vs = [c[1] for c in comps], [c[2] for c in comps]; hmax, vmax = max(hs), max(vs)
    mx, my = -(-p["w"] // (8 * hmax)), -(-p["h"] // (8 * vmax))
    if len(comps) == 1:
        mx, my = -(-p["w"] // 8), -(-p["h"] // 8)
    coef = [np.zeros((my * vs[c], mx * hs[c], 64), np.int64) for c in range(len(comps))]
    nmcu = mx * my
    ri = p["ri"] or nmcu
    segs = _segments(p["entropy"])
    for s in range(-(-nmcu // ri)):
        if s >= len(segs):
            raise EOFError("missing restart segment")
        bits, pred = _Bits(segs[s]), [0] * len(comps)
        for m in range(s * ri, min(nmcu, (s + 1) * ri)):
            by0, bx0 = divmod(m, mx)
            for ci, td, ta in scan:
                for v in range(vs[ci]):
                    for u in range(hs[ci]):
                        t = bits.huff(p["dc"][td])
                        pred[ci] += _extend(bits.get(t), t)
                        blk = np.zeros(64, np.int64); blk[0] = pred[ci]
                        k = 1
                        while k < 64:
                            rs = bits.huff(p["ac"][ta])
                            r, sz = rs >> 4, rs & 15
                            if sz:
                                k += r
                                if k > 63:
                                    raise ValueError("coefficient index past 63")
                                blk[ZIGZAG[k]] = _extend(bits.get(sz), sz); k += 1
                            elif r == 15:
                                k += 16
                            else:
                                break
                        coef[ci][by0 * vs[ci] + v, bx0 * hs[ci] + u] = blk
    return coef, hs, vs, hmax, vmax


C = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
         f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(x, shift):
    """jidctint's 1-D butterfly on the last axis (8 values), descaled by `shift` bits with rounding."""
    c = C
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * c["f0541"]
    tmp2 = z1 - z3 * c["f1847"]; tmp3 = z1 + z2 * c["f0765"]
    tmp0 = (x[..., 0] + x[..., 4]) << 13; tmp1 = (x[..., 0] - x[..., 4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * c["f1175"]
    t0, t1, t2, t3 = t0 * c["f0298"], t1 * c["f2053"], t2 * c["f3072"], t3 * c["f1501"]
    z1, z2 = -z1 * c["f0899"], -z2 * c["f2562"]
    z3, z4 = -z3 * c["f1961"] + z5, -z4 * c["f0390"] + z5
    t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4
    r = 1 << (shift - 1)
    out = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return np.stack([(o + r) >> shift for o in out], -1)


def idct_islow(coef, q):
    """[..., 64] quantised coefficients (natural order) x q[64] -> [..., 8, 8] uint8 samples."""
    blk = (coef * q).reshape(coef.shape[:-1] + (8, 8))
    ws = _idct_1d(np.swapaxes(blk, -1, -2), 11)           # columns: CONST_BITS - PASS1_BITS
    ws = np.swapaxes(ws, -1, -2)                          # ws[row, col]
    out = _idct_1d(ws, 18)                                # rows: CONST_BITS + PASS1_BITS + 3
    v = ((out & 1023) ^ 512) - 512                         # sample_range_limit's RANGE_MASK wrap
    return np.clip(v + 128, 0, 255).astype(np.uint8)


def _planes(p):
    coef, hs, vs, hmax, vmax = coefficients(p)
    out = []
    for ci, c in enumerate(coef):
        px = idct_islow(c, p["qt"][p["comps"][ci][3]])                       # [bh, bw, 8, 8]
        bh, bw = px.shape[:2]
        out.append(px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8).astype(np.int64))
    return out, hs, vs, hmax, vmax


def _fancy_h(x, wd):
    """h2v1 / h2v2 horizontal pass on rows of `wd` valid samples (edge replicated): returns (even, odd) output columns."""
    x = x[:, :wd]
    left = np.concatenate([x[:, :1], x[:, :-1]], 1)
    right = np.concatenate([x[:, 1:], x[:, -1:]], 1)
    return 3 * x + left, 3 * x + right


def upsample(plane, ch, cw, hfac, vfac, out_h, out_w):
    """jdsample: plane valid region ch x cw -> out_h x out_w (hfac, vfac in {1, 2})."""
    x = plane[:ch, :cw]
    if hfac == 1 and vfac == 1:
        return x[:out_h, :out_w]
    if cw <= 2:                                            # jinit_upsampler: fancy only when downsampled_width > 2
        x = np.repeat(np.repeat(x, hfac, 1), vfac, 0)
        return x[:out_h, :out_w]
    if vfac == 1:
        e, o = _fancy_h(x, cw)
        y = np.empty((ch, 2 * cw), np.int64)
        y[:, 0::2] = (e + 1) >> 2
        y[:, 1::2] = (o + 2) >> 2
        return y[:out_h, :out_w]
    up = np.concatenate([x[:1], x[:-1]], 0)
    dn = np.concatenate([x[1:], x[-1:]], 0)
    rows = np.empty((2 * ch, cw), np.int64)
    rows[0::2] = 3 * x + up
    rows[1::2] = 3 * x + dn
    e, o = _fancy_h(rows, cw)
    y = np.empty((2 * ch, 2 * cw), np.int64)
    y[:, 0::2] = (e + 8) >> 4
    y[:, 1::2] = (o + 7) >> 4
    return y[:out_h, :out_w]


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_rgb(Y, Cb, Cr):
    """jdcolor ycc_rgb_convert (16-bit fixed point, results clamped to 0..255)."""
    cb, cr = Cb - 128, Cr - 128
    r = Y + ((_fix(1.40200) * cr + 32768) >> 16)
    g = Y + ((-_fix(0.34414) * cb + 32768 - _fix(0.71414) * cr) >> 16)
    b = Y + ((_fix(1.77200) * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """File bytes -> uint8 [h, w, 3] RGB, bit-identical to cv2.imdecode(..., IMREAD_COLOR)[..., ::-1]."""
    p = parse(data)
    h, w = p["h"], p["w"]
    planes, hs, vs, hmax, vmax = _planes(p)
    if len(planes) == 1:
        y = planes[0][:h, :w].astype(np.uint8)
        return np.repeat(y[..., None], 3, -1)
    up = []
    for ci, pl in enumerate(planes):
        ch, cw = -(-h * vs[ci] // vmax), -(-w * hs[ci] // hmax)
        up.append(upsample(pl, ch, cw, hmax // hs[ci], vmax // vs[ci], h, w))
    return ycc_to_rgb(*up)


SIZES = [(240, 320), (142, 190), (17, 23), (1, 1)]
MODES = ["gray", 0x111111, 0x211111, 0x221111]          # cv2.IMWRITE_JPEG_SAMPLING_FACTOR: 4:4:4, 4:2:2, 4:2:0
QUALITIES = [50, 95, 100]


def textured(rng, h, w, c):
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 100 * np.sin(x / (3 + k) + y / (5 + 2 * k) + k) for k in range(c)], -1)
    return np.clip(base + rng.normal(0, 25, (h, w, c)), 0, 255).astype(np.uint8)


def corpus(h, w, seed=0):
    """Seeded cv2.imencode files of one size: every (gray / 4:4:4 / 4:2:2 / 4:2:0) x (quality 50 / 95 / 100), cycling
    through no restart markers, restart interval 1, restart interval 7 and optimised Huffman tables.  -> [(label, bytes)]."""
    import cv2
    rng = np.random.default_rng(seed * 7919 + h * 1000 + w)
    extras = [("plain", []), ("rst1", [cv2.IMWRITE_JPEG_RST_INTERVAL, 1]), ("rst7", [cv2.IMWRITE_JPEG_RST_INTERVAL, 7]),
              ("optimize", [cv2.IMWRITE_JPEG_OPTIMIZE, 1])]
    out, k = [], 0
    for mode in MODES:
        for q in QUALITIES:
            name, extra = extras[k % len(extras)]
            k += 1
            gray = mode == "gray"
            img = textured(rng, h, w, 1 if gray else 3)
            prm = [cv2.IMWRITE_JPEG_QUALITY, q] + extra + ([] if gray else [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, mode])
            ok, buf = cv2.imencode(".jpg", img[..., 0] if gray else img, prm)
            assert ok
            out.append(("%dx%d %s q%d %s" % (h, w, mode if gray else "0x%06x" % mode, q, name), buf.tobytes()))
    return out
