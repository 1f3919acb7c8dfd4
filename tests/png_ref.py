"""numpy restatement of a PNG encoder's filter stage (k4_png_encode's png_filter_kernel) and a PNG reader built on
zlib, for the tests of csrc/k4_png.cu.

The filter stage: every row of an 8-bit RGB frame (3 bytes per pixel) is filtered with each of the five PNG filters
(None, Sub, Up, Average, Paeth; PNG spec 9.2) against the previous row (zeros above row 0), and the filter with the
smallest sum of |byte as int8| over the filtered row is kept (libpng's heuristic), the lowest type on a tie."""
import struct
import zlib

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def _filters(row, prev):
    """The five filtered versions of one row, [5, 3 W] uint8."""
    x = row.astype(np.int32)
    b = prev.astype(np.int32)
    a = np.concatenate([np.zeros(3, np.int32), x[:-3]])
    c = np.concatenate([np.zeros(3, np.int32), b[:-3]])
    preds = [np.zeros_like(x), a, b, (a + b) >> 1, _paeth(a, b, c)]
    return np.stack([(x - p) & 0xff for p in preds]).astype(np.uint8)


def filter_np(frame):
    """The filtered stream of a uint8 [H, W, 3] frame: per row the filter type byte, then the filtered row."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    H, W = frame.shape[:2]
    rows = frame.reshape(H, 3 * W)
    out = np.empty((H, 1 + 3 * W), np.uint8)
    prev = np.zeros(3 * W, np.uint8)
    for y in range(H):
        f = _filters(rows[y], prev)
        s = f.view(np.int8).astype(np.int64)
        t = int(np.argmin(np.abs(s).sum(axis=1)))          # argmin: the first (lowest) type on a tie
        out[y, 0] = t
        out[y, 1:] = f[t]
        prev = rows[y]
    return out.reshape(-1)


def unfilter_np(stream, H, W):
    """The uint8 [H, W, 3] frame of a filtered stream (PNG spec 9.2, 3 bytes per pixel)."""
    s = np.asarray(stream, dtype=np.uint8).reshape(H, 1 + 3 * W)
    out = np.zeros((H, 3 * W), np.uint8)
    prev = np.zeros(3 * W, np.int32)
    for y in range(H):
        t, f = int(s[y, 0]), s[y, 1:].astype(np.int32)
        if t == 0:
            r = f
        elif t == 2:
            r = (f + prev) & 0xff
        else:                                                # Sub / Average / Paeth depend on the reconstructed left
            r = np.zeros(3 * W, np.int32)
            for i in range(3 * W):
                a = r[i - 3] if i >= 3 else 0
                c = prev[i - 3] if i >= 3 else 0
                p = a if t == 1 else (a + prev[i]) >> 1 if t == 3 else int(_paeth(np.int32(a), np.int32(prev[i]), np.int32(c)))
                r[i] = (f[i] + p) & 0xff
        if t not in (0, 1, 2, 3, 4):
            raise ValueError(f'row {y}: filter type {t}')
        out[y] = r
        prev = r
    return out.reshape(H, W, 3)


def read_png(data):
    """Parse a PNG file: checks the signature and every chunk's CRC (zlib.crc32 of type and data), returns
    ``(H, W, filtered stream, chunk types)``; ``zlib.decompress`` checks the zlib stream and its Adler-32."""
    assert data[:8] == SIGNATURE
    pos, types, idat, ihdr = 8, [], b'', None
    while pos < len(data):
        n, = struct.unpack('>I', data[pos:pos + 4])
        typ, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(typ + body), f'bad CRC in {typ}'
        types.append(typ.decode())
        if typ == b'IHDR':
            ihdr = struct.unpack('>IIBBBBB', body)
        elif typ == b'IDAT':
            idat += body
        pos += 12 + n
    assert pos == len(data) and types[0] == 'IHDR' and types[-1] == 'IEND'
    W, H, depth, ctype, comp, filt, interlace = ihdr
    assert (depth, ctype, comp, filt, interlace) == (8, 2, 0, 0, 0)
    return H, W, np.frombuffer(zlib.decompress(idat), np.uint8), types
