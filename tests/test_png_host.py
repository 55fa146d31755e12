"""CPU: the PNG container parser of monoflex_b200/png.py (chunk walk, CRCs, IHDR, zlib header) and the evaluation loader's
split reading and batch composition (monoflex_b200/loader.py). Nothing here launches: an unsupported file raises before
any call into the library."""
import io
import os
import zlib

import numpy as np
import pytest
from PIL import Image

from monoflex_b200 import png as P
from monoflex_b200.config import default_cfg
from png_util import chunk, ihdr, png_bytes, zlib_stream


def _stream():
    return zlib_stream(bytes(range(256)) * 7, 6)


@pytest.mark.parametrize("sizes", [None, [1], [1, 2, 1000], [3, 1, 1, 7]])
def test_split_idat_chunks_join_to_the_zlib_stream(sizes):
    z = _stream()
    f = P.parse_png(png_bytes(5, 2, z, idat_sizes=sizes), "x.png")
    assert (f.w, f.h, f.data) == (5, 2, z)
    assert f.filtered_bytes == 2 * 16 and f.image_bytes == 30


def test_ancillary_chunks_are_skipped():
    data = png_bytes(5, 2, _stream())
    data = data[:33] + chunk(b"tEXt", b"Comment\x00hi") + data[33:]
    assert P.parse_png(data, "x.png").data == _stream()


@pytest.mark.parametrize("where", ["IHDR", "IDAT", "IEND"])
def test_crc_errors(where):
    data = bytearray(png_bytes(5, 2, _stream(), idat_sizes=[40]))
    at = data.index(where.encode())
    data[at + 4] ^= 1 if where != "IEND" else 0          # a payload byte; IEND has none: flip its CRC
    if where == "IEND":
        data[at + 4] ^= 0x80
    with pytest.raises(ValueError, match="CRC error in the b'%s'" % where):
        P.parse_png(bytes(data), "bad.png")


@pytest.mark.parametrize("header,message", [(b"\x77\x9c", "bad zlib header"), (b"\x88\x1c", "bad zlib header"),
                                            (b"\x78\x9d", "bad zlib header"), (b"\x78\xbb", "preset dictionary"),
                                            (b"\x78", "zlib header truncated")])
def test_bad_zlib_headers(header, message):
    with pytest.raises(ValueError, match=message):
        P.parse_png(png_bytes(5, 2, header), "z.png")


def test_malformed_containers():
    good = png_bytes(5, 2, _stream())
    for data, message in ((b"GIF89a" + good[6:], "bad signature"), (good[:-12], "no IEND"),
                          (good[:-5], "truncated"), (good[:8] + good[33:], "not IHDR"),
                          (good[:8] + ihdr(5, 2) + chunk(b"IEND", b""), "no IDAT"), (png_bytes(0, 2, _stream()), "size")):
        with pytest.raises(ValueError, match=message):
            P.parse_png(data, "m.png")


def _pil_png(mode, **kw):
    buf = io.BytesIO()
    size = (6, 3)
    Image.new(mode, size).save(buf, format="PNG", **kw)
    return buf.getvalue()


@pytest.mark.parametrize("data,prop", [
    (lambda: _pil_png("L"), "colour type 0"), (lambda: _pil_png("P"), "bit depth 1"),
    (lambda: png_bytes(5, 2, _stream(), colour=3), "colour type 3"),
    (lambda: _pil_png("RGBA"), "colour type 6"), (lambda: _pil_png("LA"), "colour type 4"),
    (lambda: _pil_png("I;16"), "bit depth 16"), (lambda: _pil_png("1"), "bit depth 1"),
    (lambda: png_bytes(5, 2, _stream(), interlace=1), "interlace method 1"),
    (lambda: png_bytes(5, 2, _stream(), depth=16), "bit depth 16"),
    (lambda: png_bytes(5, 2, _stream(), compression=1), "compression method 1"),
    (lambda: png_bytes(5, 2, _stream(), filt=1), "filter method 1")])
def test_unsupported_ihdr_raises_before_any_launch(tmp_path, monkeypatch, data, prop):
    launched = []
    monkeypatch.setattr(P, "call", lambda *a: launched.append(a))
    monkeypatch.setattr(P, "DecodedImages", lambda *a: launched.append(a))
    good, bad = tmp_path / "good.png", tmp_path / "bad.png"
    good.write_bytes(png_bytes(5, 2, _stream()))
    bad.write_bytes(data())
    with pytest.raises(NotImplementedError, match="bad.png: PNG %s" % prop):
        P.decode_png([str(good), str(bad)])
    assert launched == []


@pytest.mark.parametrize("w,h", [(715827883, 1), (1, 2 ** 31 - 1), (65536, 65536), (13377, 13378), (P.MAX_PIXELS + 1, 1)])
def test_oversized_ihdr_raises_before_any_allocation_or_launch(tmp_path, monkeypatch, w, h):
    """sizes whose buffers would not fit, or would overflow 32-bit offsets, are refused on the host as PIL refuses them"""
    launched = []
    monkeypatch.setattr(P, "call", lambda *a: launched.append(a))
    monkeypatch.setattr(P, "PngBatch", lambda *a: launched.append(a))
    bad = tmp_path / "bomb.png"
    bad.write_bytes(png_bytes(w, h, zlib_stream(b"\0" * 4096, 9)))
    with pytest.raises(ValueError, match="bomb.png: image size %dx%d .* exceeds the limit of %d pixels" % (w, h, P.MAX_PIXELS)):
        P.decode_png([str(bad)])
    assert launched == []


def test_largest_accepted_size():
    f = P.parse_png(png_bytes(P.MAX_PIXELS, 1, _stream()), "wide.png")
    assert f.w * f.h == P.MAX_PIXELS and f.filtered_bytes < 2 ** 31


# ------------------------------------------------------------------------------------------------------------- loader
def make_split(root, ids, split):
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    with open(os.path.join(root, "ImageSets", split + ".txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))


@pytest.mark.parametrize("batch_size,window,expect_window", [(1, 64, 64), (3, 64, 66), (8, 64, 64), (5, 2, 5)])
def test_loader_split_and_batches(tmp_path, monkeypatch, batch_size, window, expect_window):
    from monoflex_b200 import loader as L
    monkeypatch.setattr(L, "DECODE_WINDOW", window)
    ids = ["%06d" % i for i in (7, 3, 11, 0, 5, 2, 9)]
    make_split(str(tmp_path), ids, "val")
    cfg = default_cfg()
    cfg.TEST.IMS_PER_BATCH = batch_size
    cfg.DATASETS.TEST_SPLIT = "val"
    ld = L.KittiEvalLoader(cfg, str(tmp_path))
    assert ld.dataset.ids == ids and ld.dataset.labelled and len(ld.dataset) == 7
    assert ld.dataset.imageset_txt == os.path.join(str(tmp_path), "ImageSets", "val.txt")
    assert ld.dataset.label_dir == os.path.join(str(tmp_path), "label_2")
    assert list(ld.dataset.classes) == ["Car", "Pedestrian", "Cyclist"]
    got = ld.batches()
    assert sum(got, []) == ids and all(len(b) == batch_size for b in got[:-1]) and 1 <= len(got[-1]) <= batch_size
    assert len(ld) == len(got) and ld.window == expect_window


def test_loader_test_split_and_missing_split(tmp_path):
    from monoflex_b200 import loader as L
    make_split(str(tmp_path), ["000001"], "test")
    cfg = default_cfg()
    ld = L.KittiEvalLoader(cfg, str(tmp_path))                 # default_cfg's TEST_SPLIT is "test"
    assert not ld.dataset.labelled and ld.batch_size == 1 and ld.batches() == [["000001"]]
    with pytest.raises(FileNotFoundError, match="val.txt"):
        L.KittiEvalLoader(cfg, str(tmp_path), split="val")
