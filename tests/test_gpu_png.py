"""-m gpu: the PNG decode (csrc/mf_png.cu through monoflex_b200/png.py) equals np.asarray(Image.open(f).convert('RGB'))
byte for byte, over files PIL writes, files filtered row by row with all five filter types and compressed by zlib at
every level and strategy, KITTI's widths and heights and the extremes of the deflate format (length 258, distance 1 and
32768, an empty stored block), all in one launch. Each malformed stream sets its own status, raises from check(),
writes nothing outside its buffers and leaves the other images of its launch intact."""
import io
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from monoflex_b200 import png as P
from monoflex_b200.synthetic import natural_image
from png_util import Deflate, apply_tokens, filter_rows, png_bytes, zlib_stream

pytestmark = pytest.mark.gpu
SIZES = [(1, 370), (2, 371), (3, 372), (1224, 373), (1238, 374), (1241, 375), (1242, 376)]
STRATEGIES = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE]


def pil_file(img, **kw):
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="PNG", **kw)
    return buf.getvalue()


def extremes_file():
    """an empty stored block, then fixed-Huffman blocks with a 258-byte match at distance 32768, a run of 258 at
    distance 1 and short-period references, over a 11000 x 3 image with filter type 0 on every row"""
    w, h = 11000, 3
    n = h * (1 + 3 * w)
    g = np.random.default_rng(5)
    rnd = g.integers(0, 256, n).tolist()
    row_start = set(r * (1 + 3 * w) for r in range(h))
    lit = lambda a, b: [0 if i in row_start else rnd[i] for i in range(a, b)]
    tokens = lit(0, 40000) + [(258, 32768), (258, 1), (100, 3), (7, 2)]
    pos = 40000 + 258 + 258 + 100 + 7
    tokens += lit(pos, n)
    raw = bytes(apply_tokens(tokens))
    assert len(raw) == n and all(raw[i] == 0 for i in row_start)
    d = Deflate()
    d.stored(b"")
    d.fixed(tokens[:30000])
    d.stored(b"")
    d.fixed(tokens[30000:], final=True)
    return png_bytes(w, h, d.finish(raw), idat_sizes=[1, 4096, 1, 7])


@pytest.fixture(scope="module")
def valid_files(tmp_path_factory):
    root = tmp_path_factory.mktemp("png")
    files = []
    settings = [dict(compress_level=0), dict(compress_level=1), dict(compress_level=6), dict(compress_level=9),
                dict(optimize=True)]
    k = 0
    for s in settings:
        for w, h in SIZES:
            files.append((pil_file(natural_image(w, h, k), **s), "pil_%d" % k))
            k += 1
    for level in (0, 1, 6, 9):
        for strategy in STRATEGIES:
            w, h = SIZES[k % len(SIZES)]
            raw = filter_rows(natural_image(w, h, k), [0, 1, 2, 3, 4])
            files.append((png_bytes(w, h, zlib_stream(raw, level, strategy), idat_sizes=[8192, 1, 1000]), "zlib_%d" % k))
            k += 1
    files.append((extremes_file(), "extremes"))
    paths = []
    for data, name in files:
        p = root / (name + ".png")
        p.write_bytes(data)
        paths.append(str(p))
    return paths


def pil_rgb(path):
    return np.asarray(Image.open(path).convert("RGB"))


def test_mixed_batch_equals_pil(valid_files):
    dec = P.decode_png(valid_files)
    dec.check()
    for path, img in zip(valid_files, dec.images):
        ref = pil_rgb(path)
        got = img.cpu().numpy()
        assert got.shape == ref.shape, path
        assert np.array_equal(got, ref), (path, np.argwhere(got != ref)[:5])


def test_each_setting_alone_equals_pil(valid_files):
    """the same files one launch each (a window of one image, the last lane of the grid alone)"""
    for path in valid_files[::5] + valid_files[-1:]:
        dec = P.decode_png([path])
        dec.check()
        assert np.array_equal(dec.images[0].cpu().numpy(), pil_rgb(path)), path


# ------------------------------------------------------------------------------------------------------------- malformed
W, H = 40, 6


def good_raw(seed=0):
    return filter_rows(natural_image(W, H, seed), [0, 1, 2, 3, 4])


def fixed_stream(tokens, adler_of):
    d = Deflate()
    d.fixed(tokens, final=True)
    return d.finish(adler_of)


def malformed():
    raw = good_raw()
    z = zlib_stream(raw, 6)
    over = Deflate()
    over.put(1, 1)
    over.put(2, 2)                                   # dynamic
    over.put(0, 5)
    over.put(0, 5)
    over.put(15, 4)                                  # 19 code-length codes, all of length 1: over-subscribed
    for _ in range(19):
        over.put(1, 3)
    bad_type = Deflate()
    bad_type.put(1, 1)
    bad_type.put(3, 2)
    bad_filter = bytearray(raw)
    bad_filter[2 * (1 + 3 * W)] = 5
    return [
        ("truncated", z[:len(z) // 2], 1),
        ("oversubscribed", over.finish(raw), 2),
        ("invalid_symbol", fixed_stream([raw[0], 286], raw), 2),
        ("block_type_3", bad_type.finish(raw), 3),
        ("far_distance", fixed_stream(list(raw[:5]) + [(4, 6)], raw), 4),
        ("too_long", fixed_stream(list(raw) + [1, 2, 3], raw + b"\x01\x02\x03"), 5),
        ("too_short", fixed_stream(list(raw[:-10]), raw[:-10]), 6),
        ("adler", z[:-4] + bytes([z[-4] ^ 1]) + z[-3:], 7),
        ("filter_5", zlib_stream(bytes(bad_filter), 6), 8),
    ]


def test_status_codes_are_distinct_and_named():
    assert sorted(P.STATUS) == list(range(1, 9))
    assert len(set(P.STATUS.values())) == 8


def _write(tmp_path, name, z):
    p = tmp_path / (name + ".png")
    p.write_bytes(png_bytes(W, H, z, idat_sizes=[3, 100]))
    return str(p)


def test_malformed_streams_set_their_status_and_touch_nothing_else(tmp_path):
    cases = malformed()
    good = [_write(tmp_path, "good%d" % i, zlib_stream(good_raw(i + 1), 9)) for i in range(2)]
    paths = [good[0]] + [_write(tmp_path, n, z) for n, z, _ in cases] + [good[1]]
    batch = P.PngBatch([P.read_png(p) for p in paths])
    filtered = torch.full((batch.filt_total,), 0xA5, dtype=torch.uint8, device="cuda")
    images = torch.full((batch.out_total,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((len(batch),), -1, dtype=torch.int32, device="cuda")
    batch.launch(batch.upload(), filtered, images, status)
    st = status.cpu().tolist()
    assert st == [0] + [c for _, _, c in cases] + [0], st
    for buf, offs, sizes in ((filtered, batch.filt_offsets, [p.filtered_bytes for p in batch.pngs]),
                             (images, batch.out_offsets, [p.image_bytes for p in batch.pngs])):
        outside = torch.ones(buf.numel(), dtype=torch.bool)
        for o, s in zip(offs, sizes):
            outside[o:o + s] = False
        assert bool((buf.cpu()[outside] == 0xA5).all())
    for i in (0, len(paths) - 1):
        o, p = batch.out_offsets[i], batch.pngs[i]
        got = images[o:o + p.image_bytes].view(p.h, p.w, 3).cpu().numpy()
        assert np.array_equal(got, pil_rgb(paths[i]))


def test_check_raises_naming_the_file_and_the_reason(tmp_path):
    good = _write(tmp_path, "good", zlib_stream(good_raw(), 6))
    for name, z, code in malformed():
        bad = _write(tmp_path, name, z)
        dec = P.decode_png([good, bad, good])
        with pytest.raises(ValueError, match="%s.png: PNG image data not decoded: %s" % (name, P.STATUS[code])):
            dec.check()
        assert dec.status.cpu().tolist() == [0, code, 0]
        assert np.array_equal(dec.images[2].cpu().numpy(), pil_rgb(good))


def test_staging_layout():
    """descriptor table then streams in one pinned buffer; device buffers 64-byte aligned with a gap before and after"""
    z = zlib_stream(bytes(range(256)) * 7, 6)
    files = [P.PngFile("a", 5, 2, z), P.PngFile("b", 1, 3, b"\x78\x9c\x03\x00"), P.PngFile("c", 64, 1, z)]
    b = P.PngBatch(files)
    assert b.staging.is_pinned()
    desc = b.staging.numpy()[:b.head].view(np.int64).reshape(3, P.DESC_COLS)
    assert desc[:, 1].tolist() == [len(f.data) for f in files]
    assert desc[:, 2:4].tolist() == [[5, 2], [1, 3], [64, 1]]
    for i, f in enumerate(files):
        assert b.staging.numpy()[b.head + desc[i, 0]:b.head + desc[i, 0] + desc[i, 1]].tobytes() == f.data
    for offs, sizes, total in ((b.filt_offsets, [f.filtered_bytes for f in files], b.filt_total),
                               (b.out_offsets, [f.image_bytes for f in files], b.out_total)):
        assert all(o % 64 == 0 for o in offs) and offs[0] >= 64
        ends = [o + s for o, s in zip(offs, sizes)]
        assert all(offs[i + 1] - ends[i] >= 64 for i in range(2)) and total - ends[-1] >= 64
    assert desc[:, 4].tolist() == b.filt_offsets and desc[:, 5].tolist() == b.out_offsets
