"""KITTI's PNG images decoded on the GPU: `Image.open(f).convert('RGB')` of data/datasets/kitti.py:106-114 for 8-bit RGB
non-interlaced PNGs, the only kind image_2 / image_3 hold.

    dec = decode_png(files)          # host: chunks, CRCs, headers; one H2D copy; two kernels (csrc/mf_png.cu)
    dec.check()                      # one host synchronisation; raises ValueError naming the file and the reason
    dec.images                       # uint8 [h, w, 3] CUDA tensors, bit-identical to np.asarray(Image.open(f).convert('RGB'))

This module handles the container only: the signature, the chunk walk with every CRC checked (zlib.crc32, as PIL
does), IHDR and the 2-byte zlib header. Any other PNG kind raises NotImplementedError naming the file and the property
before anything is launched. Everything inside the deflate stream is decoded - and checked - on the device."""
import struct
import zlib

import numpy as np
import torch

from ._lib import call, stream

SIGNATURE = b"\x89PNG\r\n\x1a\n"
_ALIGN = 64                      # every device buffer starts on a 64-byte boundary, with at least _ALIGN bytes between two
# PIL's DecompressionBombError bound (2 * Image.MAX_IMAGE_PIXELS): a file claiming more pixels is refused before anything
# is allocated, as PIL refuses it. KITTI's images have 0.47 M.
MAX_PIXELS = 178956970
DESC_COLS = 6                    # (src_off, src_len, w, h, filt_off, out_off), include/monoflex_b200.h
STATUS = {1: "truncated deflate stream", 2: "invalid or over-subscribed Huffman code", 3: "invalid deflate block",
          4: "back-reference before the start of the image data", 5: "more image data than the image holds",
          6: "less image data than the image holds", 7: "Adler-32 mismatch", 8: "scanline filter type above 4"}


class PngFile(object):
    """One parsed file: w, h and its zlib stream (the IDAT payloads joined)."""

    def __init__(self, name, w, h, stream_bytes):
        self.name, self.w, self.h, self.data = name, w, h, stream_bytes

    @property
    def filtered_bytes(self):
        return self.h * (1 + 3 * self.w)

    @property
    def image_bytes(self):
        return self.h * self.w * 3


def parse_png(data, name="<bytes>"):
    """The container of one PNG file's bytes -> PngFile. ValueError for a malformed file, NotImplementedError for a PNG
    kind other than 8-bit RGB non-interlaced with a zlib stream without a preset dictionary."""
    if data[:8] != SIGNATURE:
        raise ValueError("%s: not a PNG file (bad signature)" % name)
    pos, ihdr, idat, end = 8, None, [], False
    while pos < len(data):
        if pos + 8 > len(data):
            raise ValueError("%s: truncated chunk header at byte %d" % (name, pos))
        length, ctype = struct.unpack(">I4s", data[pos:pos + 8])
        if pos + 12 + length > len(data):
            raise ValueError("%s: truncated %r chunk at byte %d" % (name, ctype, pos))
        body = data[pos + 8:pos + 8 + length]
        crc = struct.unpack(">I", data[pos + 8 + length:pos + 12 + length])[0]
        if zlib.crc32(ctype + body) & 0xffffffff != crc:
            raise ValueError("%s: CRC error in the %r chunk at byte %d" % (name, ctype, pos))
        pos += 12 + length
        if ihdr is None and ctype != b"IHDR":
            raise ValueError("%s: the first chunk is %r, not IHDR" % (name, ctype))
        if ctype == b"IHDR":
            if ihdr is not None or length != 13:
                raise ValueError("%s: malformed IHDR" % name)
            ihdr = struct.unpack(">IIBBBBB", body)
            _check_ihdr(ihdr, name)
        elif ctype == b"IDAT":
            idat.append(body)
        elif ctype == b"IEND":
            end = True
            break
    if not end:
        raise ValueError("%s: no IEND chunk" % name)
    if not idat:
        raise ValueError("%s: no IDAT chunk" % name)
    z = b"".join(idat)
    if len(z) < 2:
        raise ValueError("%s: zlib header truncated" % name)
    cmf, flg = z[0], z[1]
    if cmf & 15 != 8 or cmf >> 4 > 7 or (cmf * 256 + flg) % 31:
        raise ValueError("%s: bad zlib header %02x %02x" % (name, cmf, flg))
    if flg & 0x20:
        raise ValueError("%s: zlib stream with a preset dictionary" % name)
    return PngFile(name, ihdr[0], ihdr[1], z)


def _check_ihdr(ihdr, name):
    w, h, depth, colour, compression, filt, interlace = ihdr
    if w == 0 or h == 0 or w >= 2 ** 31 or h >= 2 ** 31:
        raise ValueError("%s: image size %dx%d" % (name, w, h))
    if w * h > MAX_PIXELS:
        raise ValueError("%s: image size %dx%d (%d pixels) exceeds the limit of %d pixels, which PIL also refuses (a "
                         "possible decompression bomb)" % (name, w, h, w * h, MAX_PIXELS))
    for prop, got, want in (("bit depth", depth, 8), ("colour type", colour, 2), ("compression method", compression, 0),
                            ("filter method", filt, 0), ("interlace method", interlace, 0)):
        if got != want:
            raise NotImplementedError("%s: PNG %s %d; only 8-bit RGB non-interlaced PNGs (bit depth 8, colour type 2, "
                                      "interlace 0) are decoded" % (name, prop, got))


def read_png(path):
    with open(path, "rb") as f:
        return parse_png(f.read(), path)


IHDR_END = 33                    # signature, IHDR length and type, its 13 bytes and its CRC


def read_ihdr(path):
    """(w, h) of a PNG file from its first 33 bytes, with the signature, the IHDR CRC and the PNG kind checked as
    parse_png checks them; the rest of the file is not read."""
    with open(path, "rb") as f:
        data = f.read(IHDR_END)
    if data[:8] != SIGNATURE:
        raise ValueError("%s: not a PNG file (bad signature)" % path)
    if len(data) < IHDR_END:
        raise ValueError("%s: truncated chunk header at byte 8" % path)
    length, ctype = struct.unpack(">I4s", data[8:16])
    if ctype != b"IHDR" or length != 13:
        raise ValueError("%s: the first chunk is %r of %d bytes, not a 13-byte IHDR" % (path, ctype, length))
    if zlib.crc32(data[12:29]) & 0xffffffff != struct.unpack(">I", data[29:33])[0]:
        raise ValueError("%s: CRC error in the b'IHDR' chunk at byte 8" % path)
    ihdr = struct.unpack(">IIBBBBB", data[16:29])
    _check_ihdr(ihdr, path)
    return ihdr[0], ihdr[1]


def _aligned(sizes):
    """offsets of buffers of `sizes` bytes, each on an _ALIGN boundary with at least _ALIGN bytes before and after it;
    and the total"""
    offs, pos = [], _ALIGN
    for s in sizes:
        offs.append(pos)
        pos += (s + 2 * _ALIGN - 1) // _ALIGN * _ALIGN
    return offs, pos


def window_bytes(sizes):
    """The device bytes DecodedImages allocates for one window of images of `sizes` ((w, h) each), as PngBatch lays them
    out: (the images buffer, the filtered buffer that lives until the kernels have run)."""
    return (_aligned([w * h * 3 for w, h in sizes])[1], _aligned([h * (1 + 3 * w) for w, h in sizes])[1])


class PngBatch(object):
    """The parsed files of one decode window, staged in one pinned host buffer: the int64 descriptor table, then the zlib
    streams. filt_offsets / out_offsets and filt_total / out_total lay out the device buffers the kernels write."""

    def __init__(self, pngs):
        self.pngs = list(pngs)
        n = len(self.pngs)
        self.filt_offsets, self.filt_total = _aligned([p.filtered_bytes for p in self.pngs])
        self.out_offsets, self.out_total = _aligned([p.image_bytes for p in self.pngs])
        head = n * DESC_COLS * 8
        src_offsets, pos = [], 0
        for p in self.pngs:
            src_offsets.append(pos)
            pos += len(p.data)
        self.staging = torch.empty(head + max(pos, 1), dtype=torch.uint8, pin_memory=True)
        buf = self.staging.numpy()
        desc = buf[:head].view(np.int64).reshape(n, DESC_COLS)
        for i, p in enumerate(self.pngs):
            desc[i] = (src_offsets[i], len(p.data), p.w, p.h, self.filt_offsets[i], self.out_offsets[i])
            buf[head + src_offsets[i]:head + src_offsets[i] + len(p.data)] = np.frombuffer(p.data, dtype=np.uint8)
        self.head = head

    def __len__(self):
        return len(self.pngs)

    def upload(self, device="cuda"):
        """one asynchronous copy of the staging buffer to the device, on the current stream"""
        return self.staging.to(device, non_blocking=True)

    def launch(self, dev, filtered, images, status):
        """the two kernels on the current stream: `dev` is upload()'s buffer, filtered / images / status the device
        buffers of filt_total, out_total bytes and len(self) int32"""
        n = len(self)
        if filtered.numel() < self.filt_total or images.numel() < self.out_total or status.numel() < n:
            raise ValueError("PngBatch.launch: output buffers too small")
        desc, src = dev.data_ptr(), dev.data_ptr() + self.head
        call("mf_png_inflate", src, desc, n, filtered.data_ptr(), status.data_ptr(), stream())
        call("mf_png_unfilter", filtered.data_ptr(), desc, n, images.data_ptr(), status.data_ptr(), stream())


class DecodedImages(object):
    """The device images of one decode_png call. images: uint8 [h, w, 3] CUDA tensors (views of one buffer), status:
    int32 [n] CUDA (0 = decoded), files: the names, sizes: (w, h) per image (known from IHDR before the decode)."""

    def __init__(self, batch, device):
        dev = torch.device(device)
        self.files = [p.name for p in batch.pngs]
        self.sizes = [(p.w, p.h) for p in batch.pngs]
        self.buffer = torch.empty(batch.out_total, dtype=torch.uint8, device=dev)
        filtered = torch.empty(batch.filt_total, dtype=torch.uint8, device=dev)
        self.status = torch.empty(len(batch), dtype=torch.int32, device=dev)
        staged = batch.upload(dev)
        batch.launch(staged, filtered, self.buffer, self.status)
        self._status_host = torch.empty(len(batch), dtype=torch.int32).pin_memory()
        self._status_host.copy_(self.status, non_blocking=True)
        self.event = torch.cuda.Event()
        self.event.record()
        self.images = [self.buffer[o:o + p.image_bytes].view(p.h, p.w, 3) for o, p in zip(batch.out_offsets, batch.pngs)]
        self._keep = (batch, staged, filtered)           # alive until the kernels have run (stream ordered)

    def __len__(self):
        return len(self.images)

    def check(self):
        """Raise ValueError naming the first file that did not decode and why. Waits for this decode only (one host
        synchronisation on its event)."""
        self.event.synchronize()
        for name, s in zip(self.files, self._status_host.tolist()):
            if s:
                raise ValueError("%s: PNG image data not decoded: %s (status %d)" % (name, STATUS.get(s, "unknown"), s))


def decode_png(files, device="cuda"):
    """Decode a window of PNG files (paths) on the current CUDA stream. Every file is parsed and checked on the host
    before anything is launched; nothing here waits for the device."""
    return DecodedImages(PngBatch([read_png(f) for f in files]), device)
