"""NumPy restatement of the baseline-JPEG encoder of csrc/jpeg_enc.cu (test infrastructure only, like oracle/jpeg.py).

Encodes uint8 BGR [h,w,3] (YCbCr 4:2:0) or gray [h,w] the way cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) does
with libjpeg-turbo's defaults:
  markers     SOI, APP0 JFIF 1.01 (no density unit, 1:1), DQT per table, SOF0, DHT per table (DC0, AC0, DC1, AC1; the
              standard tables), SOS, entropy-coded data, EOI; no restart markers.
  quality     jpeg_set_quality(q, force_baseline=TRUE): scale 5000/q below 50, else 200 - 2q; (t*scale + 50) / 100
              clamped to 1..255.
  colour      jccolor.c rgb_ycc: 16-bit fixed point, ONE_HALF rounding for Y, ONE_HALF - 1 for Cb / Cr.
  downsample  jcsample.c h2v2: 2x2 sums with a bias alternating 1, 2 along each output row; columns replicated to whole
              MCUs by the downsampler, rows by the prep controller (the last converted row pair, then the last chroma row).
  DCT         jfdctint.c ISLOW (CONST_BITS 13, PASS1_BITS 2) on samples - 128.
  quantise    jcdctmgr.c compute_reciprocal / quantize: (|x| + corr) * recip >> (16 + shift), sign restored, divisor q << 3.
  entropy     standard tables; DC differences per component; ZRL / EOB; 0xFF stuffed with 0x00; final byte padded
              with 1-bits.  Dummy blocks (jccoefct.c compress_data): luma blocks of the last MCU column / row that lie
              outside the component are zero-AC blocks carrying the DC of the block before them.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63])

STD_LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                       49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_Q = np.full(64, 99, np.int64)
STD_CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# jstdhuff.c: (bits[1..16], values) of DC luma, AC luma, DC chroma, AC chroma
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16,
    0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6,
    0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8,
    0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34,
    0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4,
    0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6,
    0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])


def huff_codes(table):
    """(bits, values) -> {symbol: (code, length)}: jchuff.c jpeg_make_c_derived_tbl's canonical code assignment."""
    bits, vals = table
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


def quant_tables(quality):
    """jpeg_set_quality(quality, TRUE): the luma and chroma tables (natural order, int64)."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((t * scale + 50) // 100, 1, 255) for t in (STD_LUMA_Q, STD_CHROMA_Q)]


def reciprocal(divisor):
    """jcdctmgr.c compute_reciprocal with 16-bit DCTELEM: (recip, corr, shift)."""
    b = int(divisor).bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, int(divisor))
    c = int(divisor) // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= int(divisor) // 2:
        c += 1
    else:
        fq += 1
    return fq, c, r - 16


def header(h, w, channels, quality):
    """Every byte before the entropy-coded data."""
    def seg(marker, payload):
        return bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + bytes(payload)
    qt = quant_tables(quality)
    nt = 2 if channels == 3 else 1
    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(nt):
        out += seg(0xDB, [t] + [int(v) for v in qt[t][ZIGZAG]])
    comps = [(1, 0x22 if channels == 3 else 0x11, 0), (2, 0x11, 1), (3, 0x11, 1)][:channels]
    out += seg(0xC0, [8, h >> 8, h & 255, w >> 8, w & 255, channels] + [v for c in comps for v in c])
    for t in range(nt):
        for cls, tab in ((0, (DC_LUMA, DC_CHROMA)[t]), (1, (AC_LUMA, AC_CHROMA)[t])):
            out += seg(0xC4, [cls << 4 | t] + tab[0] + tab[1])
    out += seg(0xDA, [channels] + [v for c in range(channels) for v in (c + 1, 0x00 if c == 0 else 0x11)] + [0, 63, 0])
    return out


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc(bgr):
    """uint8 [h,w,3] BGR -> int64 Y, Cb, Cr planes (jccolor.c)."""
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    half = 1 << 15
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + (128 << 16) + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + (128 << 16) + half - 1) >> 16
    return y, cb, cr


def downsample_h2v2(plane, h, w):
    """Full-resolution plane [h,w] -> chroma plane [8*ceil(h/16), 8*ceil(w/16)]."""
    ch, cw = 8 * ((h + 15) // 16), 8 * ((w + 15) // 16)
    cols = np.minimum(np.arange(2 * cw), w - 1)
    rows = np.minimum(np.arange(2 * ((h + 1) // 2)), h - 1)             # the colour buffer pads the last row pair
    p = plane[rows][:, cols]
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    s = (s + np.where(np.arange(cw) % 2 == 0, 1, 2)[None, :]) >> 2
    return s[np.minimum(np.arange(ch), s.shape[0] - 1)]                   # then the last chroma row is replicated


def pad_plane(plane, ph, pw):
    h, w = plane.shape
    return plane[np.minimum(np.arange(ph), h - 1)][:, np.minimum(np.arange(pw), w - 1)]


def fdct_islow(blocks):
    """int64 [..., 8, 8] samples - 128 -> jfdctint.c output (scaled by 8), int64 [..., 8, 8]."""
    F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
             f2053=16819, f2562=20995, f3072=25172)

    def descale(x, n):
        return (x + (1 << (n - 1))) >> n

    def one_pass(d, axis, first):
        d = np.moveaxis(d, axis, -1)
        x = [d[..., i] for i in range(8)]
        t0, t7 = x[0] + x[7], x[0] - x[7]
        t1, t6 = x[1] + x[6], x[1] - x[6]
        t2, t5 = x[2] + x[5], x[2] - x[5]
        t3, t4 = x[3] + x[4], x[3] - x[4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        o = [None] * 8
        sh = 13 - 2 if first else 13 + 2
        if first:
            o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
        else:
            o[0], o[4] = descale(t10 + t11, 2), descale(t10 - t11, 2)
        z1 = (t12 + t13) * F["f0541"]
        o[2] = descale(z1 + t13 * F["f0765"], sh)
        o[6] = descale(z1 - t12 * F["f1847"], sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * F["f1175"]
        t4, t5, t6, t7 = t4 * F["f0298"], t5 * F["f2053"], t6 * F["f3072"], t7 * F["f1501"]
        z1, z2 = z1 * -F["f0899"], z2 * -F["f2562"]
        z3, z4 = z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
        o[7] = descale(t4 + z1 + z3, sh)
        o[5] = descale(t5 + z2 + z4, sh)
        o[3] = descale(t6 + z2 + z3, sh)
        o[1] = descale(t7 + z1 + z4, sh)
        return np.moveaxis(np.stack(o, -1), -1, axis)

    return one_pass(one_pass(blocks, -1, True), -2, False)


def quantize(coefs, qt):
    """ISLOW output [..., 64] natural order, table [64] -> quantised int64 [..., 64]."""
    rq = np.array([reciprocal(int(q) << 3) for q in qt], np.int64)
    a = np.abs(coefs)
    v = ((a + rq[:, 1]) * rq[:, 0]) >> (16 + rq[:, 2])
    return np.where(coefs < 0, -v, v)


def plane_blocks(plane, qt):
    """Padded sample plane [8*bh, 8*bw] -> quantised coefficients [bh, bw, 64] (natural order)."""
    ph, pw = plane.shape
    b = (plane - 128).reshape(ph // 8, 8, pw // 8, 8).transpose(0, 2, 1, 3)
    return quantize(fdct_islow(b).reshape(ph // 8, pw // 8, 64), qt)


class _Bits:
    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, code, length):
        self.acc = (self.acc << length) | code
        self.n += length


def _nbits(v):
    return int(abs(int(v))).bit_length()


def _block(bits, zz, pred, dct, act):
    """One block (coefficients in zigzag order, DC first); returns the DC for the next prediction."""
    diff = int(zz[0]) - pred
    nb = _nbits(diff)
    bits.put(*dct[nb])
    if nb:
        bits.put((diff if diff >= 0 else diff - 1) & ((1 << nb) - 1), nb)
    nz = np.flatnonzero(zz[1:]) + 1
    last = 0
    for k in nz:
        r = int(k) - last - 1
        while r > 15:
            bits.put(*act[0xF0])
            r -= 16
        v = int(zz[k])
        nb = _nbits(v)
        bits.put(*act[(r << 4) | nb])
        bits.put((v if v >= 0 else v - 1) & ((1 << nb) - 1), nb)
        last = int(k)
    if last < 63:
        bits.put(*act[0x00])
    return int(zz[0])


def encode(img, quality=95):
    """uint8 [h,w,3] BGR or [h,w] gray -> bytes, equal to cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality])[1]."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim in (2, 3)
    h, w = img.shape[:2]
    channels = 3 if img.ndim == 3 else 1
    qt = quant_tables(quality)
    codes = [(huff_codes(DC_LUMA), huff_codes(AC_LUMA)), (huff_codes(DC_CHROMA), huff_codes(AC_CHROMA))]
    bits = _Bits()
    if channels == 1:
        bh, bw = (h + 7) // 8, (w + 7) // 8
        Y = plane_blocks(pad_plane(img.astype(np.int64), 8 * bh, 8 * bw), qt[0])[..., ZIGZAG]
        pred = 0
        for by in range(bh):
            for bx in range(bw):
                pred = _block(bits, Y[by, bx], pred, *codes[0])
    else:
        y, cb, cr = ycc(img)
        bh, bw = (h + 7) // 8, (w + 7) // 8                              # luma blocks inside the component
        mh, mw = (h + 15) // 16, (w + 15) // 16                          # MCUs
        Y = plane_blocks(pad_plane(y, 8 * bh, 8 * bw), qt[0])[..., ZIGZAG]
        C = [plane_blocks(downsample_h2v2(p, h, w), qt[1])[..., ZIGZAG] for p in (cb, cr)]
        eob = np.zeros(64, np.int64)
        pred = [0, 0, 0]
        for my in range(mh):
            for mx in range(mw):
                mcu = []
                for v in range(2):
                    for u in range(2):
                        by, bx = 2 * my + v, 2 * mx + u
                        if by >= bh:                                     # a dummy row: DC of the MCU's previous block
                            blk = eob.copy(); blk[0] = mcu[-1][0]
                        elif bx >= bw:                                   # a dummy column: DC of the block to its left
                            blk = eob.copy(); blk[0] = mcu[-1][0]
                        else:
                            blk = Y[by, bx]
                        mcu.append(blk)
                for blk in mcu:
                    pred[0] = _block(bits, blk, pred[0], *codes[0])
                for c in (1, 2):
                    pred[c] = _block(bits, C[c - 1][my, mx], pred[c], *codes[1])
    pad = (-bits.n) % 8
    bits.put((1 << pad) - 1, pad)
    raw = bits.acc.to_bytes(bits.n // 8, "big") if bits.n else b""
    return header(h, w, channels, quality) + raw.replace(b"\xff", b"\xff\x00") + b"\xff\xd9"


SIZES = [(240, 320), (142, 190), (480, 640), (17, 23), (9, 9), (8, 16), (16, 8), (1, 1)]
QUALITIES = [1, 10, 50, 75, 95, 100]
KINDS = ["texture", "noise", "zeros", "full", "checker", "gradient"]


def image(kind, h, w, channels, seed=0):
    """One seeded test image: a smooth texture, uniform noise (long codes, many 0xFF bytes), constant 0 / 255, a
    checkerboard of 3-pixel squares, or a gradient; uint8 [h,w,3] BGR or [h,w]."""
    rng = np.random.default_rng(seed)
    shape = (h, w, channels)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    if kind == "noise":
        img = rng.integers(0, 256, shape)
    elif kind == "zeros":
        img = np.zeros(shape)
    elif kind == "full":
        img = np.full(shape, 255)
    elif kind == "checker":
        img = np.repeat((((yy // 3 + xx // 3) % 2) * 255)[..., None], channels, -1)
        if channels == 3:
            img[..., 2] = 255 - img[..., 2]
    elif kind == "gradient":
        img = np.stack([(yy * 7 + xx * 3 + 40 * c) % 256 for c in range(channels)], -1)
    else:
        ph = rng.uniform(0, 2 * np.pi, (channels, 3))
        img = np.stack([128 + 60 * np.sin(xx / 7.0 + ph[c, 0]) * np.cos(yy / 11.0 + ph[c, 1]) + 40 * np.sin((xx + yy) / 3.0 + ph[c, 2])
                        for c in range(channels)], -1) + rng.normal(0, 6, shape)
    img = np.clip(img, 0, 255).astype(np.uint8)
    return img if channels == 3 else img[..., 0]


def corpus(h, w, channels):
    """[(label, image, quality)] of one size: every kind at quality 95, and the texture and noise at every quality."""
    out = [("%s-q95" % k, image(k, h, w, channels, seed=i), 95) for i, k in enumerate(KINDS)]
    for q in QUALITIES:
        if q != 95:
            out += [("%s-q%d" % (k, q), image(k, h, w, channels, seed=100 + q), q) for k in ("texture", "noise")]
    return out


def capacity(h, w, channels):
    """Worst-case file size (udh_jpeg_encode_capacity): the header, every block at its longest code (the DC at 11 bits of
    category 11 plus its longest code, 63 AC coefficients at 16 + 10 bits) with every byte stuffed, and EOI."""
    if channels == 3:
        nblk = 6 * ((h + 15) // 16) * ((w + 15) // 16)
    else:
        nblk = ((h + 7) // 8) * ((w + 7) // 8)
    return len(header(h, w, channels, 95)) + 2 * ((nblk * (11 + 11 + 63 * 26) + 7) // 8) + 2
