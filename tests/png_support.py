"""A small PNG encoder on the standard library (zlib, struct, binascii.crc32) and NumPy, for writing test images without OpenCV.

It covers what the decoder in csrc/icc_png.hpp reads: colour types 0, 2, 3, 4 and 6 at every bit depth the format allows, any of the five
row filters per row, Adam7 interlacing, IDAT split into several chunks, PLTE / tRNS, and extra chunks passed through as given."""
import binascii
import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]   # (x0, y0, dx, dy)


def chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", binascii.crc32(kind + data) & 0xFFFFFFFF)


def _rows(samples, bit_depth):
    """(h, w, c) integer samples -> (h, row bytes) uint8: big-endian 16-bit samples, or sub-byte samples packed from the high bits."""
    s = np.asarray(samples).astype(np.uint32)
    h, w, c = s.shape
    if bit_depth == 16:
        return s.astype(">u2").view(np.uint8).reshape(h, w * c * 2)
    if bit_depth == 8:
        return s.astype(np.uint8).reshape(h, w * c)
    per = 8 // bit_depth
    flat = s.reshape(h, w * c)
    n = (w * c + per - 1) // per
    pad = np.zeros((h, n * per), np.uint32)
    pad[:, :w * c] = flat
    pad = pad.reshape(h, n, per)
    shifts = np.array([8 - bit_depth * (k + 1) for k in range(per)], np.uint32)
    return (pad << shifts).sum(-1).astype(np.uint8)


def _filter(raw, bpp, kinds):
    """Filtered scanlines (each prefixed by its filter byte) of raw (h, n) uint8 rows; kinds: one filter type per row."""
    x = raw.astype(np.int32)
    h, n = x.shape
    prior = np.zeros_like(x)
    prior[1:] = x[:-1]
    left = np.zeros_like(x)
    left[:, bpp:] = x[:, :-bpp]
    upleft = np.zeros_like(x)
    upleft[:, bpp:] = prior[:, :-bpp]
    kinds = np.asarray(kinds, np.int64)
    out = np.zeros((h, n + 1), np.int32)
    out[:, 0] = kinds
    for k in np.unique(kinds):
        r = kinds == k
        if k == 0:
            f = x[r]
        elif k == 1:
            f = x[r] - left[r]
        elif k == 2:
            f = x[r] - prior[r]
        elif k == 3:
            f = x[r] - (left[r] + prior[r]) // 2
        else:
            a, b, c = left[r], prior[r], upleft[r]
            p = a + b - c
            pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
            f = x[r] - np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        out[r, 1:] = f & 0xFF
    return out.astype(np.uint8).tobytes()


def encode_png(samples, color_type: int, bit_depth: int = 8, filters=4, interlace: bool = False, level: int = 6, idat_chunks: int = 1,
               palette=None, trns: bytes = None, extra_chunks=(), after_idat=()) -> bytes:
    """PNG bytes of `samples`: (h, w) for colour types 0 and 3 (palette indices), (h, w, c) otherwise, in the file's channel order
    (R, G, B[, A], or gray[, alpha]) and value range.  filters: one type for every row, or a callable (pass, row) -> type.
    palette: (n, 3) RGB entries for colour type 3.  extra_chunks: (type, data) written before IDAT; after_idat: after it."""
    s = np.asarray(samples)
    if s.ndim == 2:
        s = s[:, :, None]
    h, w, c = s.shape
    assert c == CHANNELS[color_type], (c, color_type)
    bpp = max(1, c * bit_depth // 8)
    pick = filters if callable(filters) else (lambda p, y: filters)
    body = []
    passes = ADAM7 if interlace else [(0, 0, 1, 1)]
    for k, (x0, y0, dx, dy) in enumerate(passes):
        sub = s[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        body.append(_filter(_rows(sub, bit_depth), bpp, [pick(k, y) for y in range(sub.shape[0])]))
    z = zlib.compress(b"".join(body), level)
    out = [SIGNATURE, chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bit_depth, color_type, 0, 0, 1 if interlace else 0))]
    if palette is not None:
        out.append(chunk(b"PLTE", np.asarray(palette, np.uint8).reshape(-1).tobytes()))
    if trns is not None:
        out.append(chunk(b"tRNS", trns))
    out += [chunk(t, d) for t, d in extra_chunks]
    cuts = np.linspace(0, len(z), idat_chunks + 1).astype(int)
    out += [chunk(b"IDAT", z[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    out += [chunk(t, d) for t, d in after_idat]
    out.append(chunk(b"IEND", b""))
    return b"".join(out)


def write_png(path: str, img, level: int = 1, filters=4) -> None:
    """An 8-bit image as cv2.imwrite would hand it over: (h, w) gray, or (h, w, 3) in B, G, R order (stored as RGB)."""
    a = np.asarray(img, np.uint8)
    data = encode_png(a, 0, 8, filters, level=level) if a.ndim == 2 else encode_png(a[:, :, ::-1], 2, 8, filters, level=level)
    with open(path, "wb") as f:
        f.write(data)
