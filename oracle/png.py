"""NumPy / zlib restatement of the PNG decoder of csrc/png.cu (test infrastructure only, like oracle/jpeg.py), and the test
PNG files.

parse() walks the chunks as the library's host parser does and returns its reason codes (_lib.PNG_R); decode() inflates
the IDAT stream with zlib.decompress, undoes the five row filters and returns what cv2.imread(..., IMREAD_COLOR) returns
for the files the parser accepts: uint8 [h, w, 3] BGR, gray replicated, alpha dropped.  The filters of rows that need
the reconstructed left neighbour (Sub, Average, Paeth) run as a plain per-byte loop: slow, but only tests run it.
"""
import struct
import zlib

import numpy as np

from oracle import jpeg as J

SIG = b"\x89PNG\r\n\x1a\n"
R = dict(OK=0, NOT_PNG=1, JPEG=2, TRUNCATED=3, IDAT_TRUNCATED=4, CRC=5, NO_IEND=6, MALFORMED=7, PALETTE=8, DEPTH16=9,
         DEPTH_SUB8=10, INTERLACED=11, GRAY_ALPHA=12, CHUNK=13)
IGNORED = (b"tEXt", b"zTXt", b"iTXt", b"tIME", b"pHYs")   # ancillary chunks cv2.imread(IMREAD_COLOR) does not act on
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
VALID_DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}


def parse(data):
    """-> (reason, dict(width, height, bit_depth, color_type, interlace, channels), zlib stream bytes)."""
    info, idat = {}, []
    if data[:3] == b"\xff\xd8\xff":
        return R["JPEG"], info, b""
    if data[:8] != SIG:
        return R["NOT_PNG"], info, b""
    pos, iend, other, closed = 8, False, False, False
    while pos < len(data):
        if len(data) - pos < 8:
            return R["TRUNCATED"], info, b""
        n, typ = struct.unpack(">I", data[pos:pos + 4])[0], data[pos + 4:pos + 8]
        if n > 0x7fffffff:
            return R["MALFORMED"], info, b""
        if n + 12 > len(data) - pos:
            return R["IDAT_TRUNCATED" if typ == b"IDAT" else "TRUNCATED"], info, b""
        body = data[pos + 8:pos + 8 + n]
        if zlib.crc32(typ + body) != struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]:
            return R["CRC"], info, b""
        if not info:
            if typ != b"IHDR" or n != 13:
                return R["MALFORMED"], info, b""
            w, h, depth, ct, comp, filt, il = struct.unpack(">IIBBBBB", body)
            if not (0 < w <= 0x7fffffff and 0 < h <= 0x7fffffff) or comp or filt or il > 1 or depth not in VALID_DEPTHS.get(ct, ()):
                return R["MALFORMED"], info, b""
            info = dict(width=w, height=h, bit_depth=depth, color_type=ct, interlace=il, channels=CHANNELS[ct])
        elif typ == b"IDAT":
            if closed:
                return R["MALFORMED"], info, b""
            idat.append(body)
        elif typ == b"IEND":
            iend = True
            break
        elif typ == b"IHDR":
            return R["MALFORMED"], info, b""
        elif typ not in IGNORED:
            other = True
        closed = closed or (bool(idat) and typ != b"IDAT")
        pos += n + 12
    if not iend:
        return R["NO_IEND"], info, b""
    if not info or not idat:
        return R["MALFORMED"], info, b""
    for cond, reason in ((info["color_type"] == 3, "PALETTE"), (info["bit_depth"] == 16, "DEPTH16"), (info["bit_depth"] < 8, "DEPTH_SUB8"),
                         (info["interlace"], "INTERLACED"), (info["color_type"] == 4, "GRAY_ALPHA"), (other, "CHUNK")):
        if cond:
            return R[reason], info, b""
    return R["OK"], info, b"".join(idat)


def unfilter(raw, h, w, bpp):
    """Filtered scanlines (h rows of 1 + w * bpp bytes) -> uint8 [h, w * bpp]."""
    rb = w * bpp
    rows = np.frombuffer(raw, np.uint8).reshape(h, rb + 1)
    out = np.zeros((h, rb), np.uint8)
    prev = np.zeros(rb, np.int64)
    for y in range(h):
        f, cur = int(rows[y, 0]), rows[y, 1:].astype(np.int64)
        if f == 0:
            rec = cur
        elif f == 2:
            rec = (cur + prev) & 255
        elif f in (1, 3, 4):
            c, p, rec = cur.tolist(), prev.tolist(), [0] * rb
            for i in range(rb):
                a = rec[i - bpp] if i >= bpp else 0
                b = p[i]
                cc = p[i - bpp] if i >= bpp else 0
                if f == 1:
                    pred = a
                elif f == 3:
                    pred = (a + b) >> 1
                else:
                    pa, pb, pc = abs(b - cc), abs(a - cc), abs(a + b - 2 * cc)
                    pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else cc)
                rec[i] = (c[i] + pred) & 255
            rec = np.array(rec, np.int64)
        else:
            raise ValueError("unknown filter type %d in row %d" % (f, y))
        out[y] = rec
        prev = rec
    return out


def decode(data):
    """cv2.imread(..., IMREAD_COLOR) of a file the parser accepts: uint8 [h, w, 3] BGR."""
    reason, info, stream = parse(data)
    if reason:
        raise ValueError("not a file the device decoder takes (reason %d)" % reason)
    h, w, ch = info["height"], info["width"], info["channels"]
    raw = zlib.decompress(stream)
    if len(raw) != h * (1 + w * ch):
        raise ValueError("%d bytes of scanlines, %d expected" % (len(raw), h * (1 + w * ch)))
    px = unfilter(raw, h, w, ch).reshape(h, w, ch)
    if ch == 1:
        return np.repeat(px, 3, axis=2)
    return np.ascontiguousarray(px[..., 2::-1])


# ---- test files ---------------------------------------------------------------------------------------------------------
def chunk(typ, body):
    return struct.pack(">I", len(body)) + typ + body + struct.pack(">I", zlib.crc32(typ + body))


def ihdr(h, w, depth=8, color_type=2, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color_type, 0, 0, interlace))


def filter_rows(px, filters):
    """uint8 [h, w, ch] pixels and one filter type per row -> the filtered scanlines (bytes)."""
    h, w, ch = px.shape
    rows = px.reshape(h, w * ch).astype(np.int64)
    out = []
    for y in range(h):
        x = rows[y]
        b = rows[y - 1] if y else np.zeros_like(x)
        a = np.concatenate([np.zeros(ch, np.int64), x[:-ch]])
        c = np.concatenate([np.zeros(ch, np.int64), b[:-ch]])
        f = filters[y]
        if f == 0:
            pred = np.zeros_like(x)
        elif f == 1:
            pred = a
        elif f == 2:
            pred = b
        elif f == 3:
            pred = (a + b) >> 1
        else:
            pa, pb, pc = np.abs(b - c), np.abs(a - c), np.abs(a + b - 2 * c)
            pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        out.append(bytes([f]) + ((x - pred) & 255).astype(np.uint8).tobytes())
    return b"".join(out)


def make_png(px, filters, level=6, idat_split=0, extra=(), stream=None):
    """A PNG of uint8 [h, w, ch] pixels (ch 1: gray, 3: RGB, 4: RGBA, in the file's own channel order) with the given row
    filters, compressed by zlib at `level`; idat_split > 0 cuts the stream into IDAT chunks of that many bytes; `extra`
    chunks go before the first IDAT; `stream` replaces the zlib stream."""
    h, w, ch = px.shape
    z = stream if stream is not None else zlib.compress(filter_rows(px, filters), level)
    parts = [z[i:i + idat_split] for i in range(0, len(z), idat_split)] if idat_split else [z]
    return SIG + ihdr(h, w, 8, {1: 0, 3: 2, 4: 6}[ch]) + b"".join(extra) + b"".join(chunk(b"IDAT", p) for p in parts) + chunk(b"IEND", b"")


SIZES = [(17, 23), (1, 37), (29, 1), (1, 1), (64, 50)]
LEVELS = [0, 1, 6, 9]


def textured(rng, h, w, c):
    return J.textured(rng, h, w, c)


def corpus(h, w, seed=0):
    """(label, file bytes) pairs of one size: cv2.imencode at compression levels 0, 1, 6 and 9 (stored, fixed and dynamic
    blocks; cv2's run-length strategy and zlib's default one) for gray, BGR and BGRA images, and zlib files whose rows use
    every filter type (each type on every row, and a seeded mix), split over several IDAT chunks."""
    import cv2
    rng = np.random.default_rng(seed)
    out = []
    for c in (1, 3, 4):
        img = textured(rng, h, w, c if c != 4 else 3)
        if c == 4:
            img = np.concatenate([img, rng.integers(0, 256, (h, w, 1), dtype=np.uint8)], axis=2)
        src = img[..., 0] if c == 1 else img
        for level in LEVELS:
            for strategy in ((None, cv2.IMWRITE_PNG_STRATEGY_DEFAULT) if level == 9 else (None,)):
                prm = [cv2.IMWRITE_PNG_COMPRESSION, level] + ([cv2.IMWRITE_PNG_STRATEGY, strategy] if strategy is not None else [])
                ok, buf = cv2.imencode(".png", src, prm)
                assert ok
                out.append(("cv2-c%d-l%d%s" % (c, level, "-default" if strategy is not None else ""), buf.tobytes()))
        px = img[..., ::-1] if c >= 3 else img             # the file's channel order: RGB(A)
        if c == 4:
            px = np.concatenate([img[..., 2::-1], img[..., 3:]], axis=2)
        for f in range(5):
            out.append(("zlib-c%d-f%d" % (c, f), make_png(px, [f] * h, level=6, idat_split=97)))
        out.append(("zlib-c%d-mix" % c, make_png(px, rng.integers(0, 5, h).tolist(), level=9, idat_split=1000)))
    flat = np.zeros((h, w, 3), np.uint8)
    flat[:] = [7, 7, 7]
    out.append(("zlib-flat-l1", make_png(flat, [0] * h, level=1)))     # long runs: matches that overlap their own output
    return out
