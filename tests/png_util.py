"""PNG fixtures made at test time: a chunk writer, a row-filtering encoder over
zlib.compressobj, and a deflate writer whose blocks and tokens the test chooses (for matches zlib never emits, such as a
distance of 32768, and for malformed streams)."""
import struct
import zlib

import numpy as np


def chunk(ctype, body):
    return struct.pack(">I", len(body)) + ctype + body + struct.pack(">I", zlib.crc32(ctype + body) & 0xffffffff)


def ihdr(w, h, depth=8, colour=2, compression=0, filt=0, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, colour, compression, filt, interlace))


def png_bytes(w, h, zstream, idat_sizes=None, **ihdr_kw):
    """a PNG file around `zstream`, split into IDAT chunks of idat_sizes (cycled; None: one chunk)"""
    parts, pos, k = [], 0, 0
    while pos < len(zstream) or not parts:
        n = len(zstream) - pos if idat_sizes is None else idat_sizes[k % len(idat_sizes)]
        parts.append(chunk(b"IDAT", zstream[pos:pos + n]))
        pos += n
        k += 1
    return b"\x89PNG\r\n\x1a\n" + ihdr(w, h, **ihdr_kw) + b"".join(parts) + chunk(b"IEND", b"")


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(img, types):
    """PNG's forward filters, row r with filter types[r % len(types)] -> the filtered scanlines (bytes)"""
    h, w, _ = img.shape
    px = img.reshape(h, w * 3).astype(np.int32)
    out = bytearray()
    for r in range(h):
        ft = types[r % len(types)]
        cur = px[r]
        up = px[r - 1] if r else np.zeros_like(cur)
        left = np.concatenate([np.zeros(3, np.int32), cur[:-3]])
        ul = np.concatenate([np.zeros(3, np.int32), up[:-3]])
        pred = {0: 0, 1: left, 2: up, 3: (left + up) >> 1, 4: _paeth(left, up, ul)}[ft]
        out.append(ft)
        out += ((cur - pred) & 255).astype(np.uint8).tobytes()
    return bytes(out)


def zlib_stream(raw, level, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return c.compress(raw) + c.flush()


class Deflate(object):
    """A deflate writer: stored and fixed-Huffman blocks of chosen tokens, raw bits for anything else."""

    def __init__(self):
        self.bits, self.n = 0, 0
        self.out = bytearray()

    def put(self, value, nbits):                        # LSB-first
        self.bits |= value << self.n
        self.n += nbits
        while self.n >= 8:
            self.out.append(self.bits & 255)
            self.bits >>= 8
            self.n -= 8

    def put_code(self, code, nbits):                    # Huffman codes are packed MSB-first
        self.put(int(format(code, "0%db" % nbits)[::-1], 2), nbits)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def stored(self, data, final=False):
        self.put(1 if final else 0, 1)
        self.put(0, 2)
        self.align()
        self.put(len(data), 16)
        self.put(len(data) ^ 0xffff, 16)
        self.out += data

    def fixed_sym(self, s):
        if s < 144:
            self.put_code(0x30 + s, 8)
        elif s < 256:
            self.put_code(0x190 + s - 144, 9)
        elif s < 280:
            self.put_code(s - 256, 7)
        else:
            self.put_code(0xc0 + s - 280, 8)

    def fixed(self, tokens, final=False):
        """tokens: ints (literals) or (length, distance) pairs"""
        self.put(1 if final else 0, 1)
        self.put(1, 2)
        for t in tokens:
            if isinstance(t, tuple):
                length, dist = t
                base = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163,
                        195, 227, 258]
                extra = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
                i = 28 if length == 258 else max(k for k in range(28) if base[k] <= length)
                self.fixed_sym(257 + i)
                self.put(length - base[i], extra[i])
                dbase = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049,
                         3073, 4097, 6145, 8193, 12289, 16385, 24577]
                dextra = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
                j = max(k for k in range(30) if dbase[k] <= dist)
                self.put_code(j, 5)
                self.put(dist - dbase[j], dextra[j])
            else:
                self.fixed_sym(t)
        self.fixed_sym(256)

    def finish(self, adler_of):
        """the zlib stream: header, the blocks written so far, Adler-32 of `adler_of`"""
        self.align()
        return b"\x78\x9c" + bytes(self.out) + struct.pack(">I", zlib.adler32(adler_of) & 0xffffffff)


def apply_tokens(tokens, out=None):
    """the bytes a token list produces (what an inflater writes)"""
    out = bytearray() if out is None else out
    for t in tokens:
        if isinstance(t, tuple):
            length, dist = t
            for _ in range(length):
                out.append(out[-dist])
        else:
            out.append(t)
    return out
