"""Host-only checks of the GPU JPEG decoder's parser (gp_jpeg_probe): what it takes, what it leaves to Pillow, and
clean rejection of malformed headers."""
import io
import os

import numpy as np
import pytest
from PIL import Image

from genpercept_b200 import engine as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def encode(h, w, mode="RGB", **kw):
    g = np.random.default_rng(h * 13 + w)
    a = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    im = Image.fromarray(a).convert(mode)
    buf = io.BytesIO()
    im.save(buf, "JPEG", **kw)
    return buf.getvalue()


def segment(d, marker):
    """Offset of the first marker segment `marker` (0xFFxx) in the header."""
    i = 2
    while i + 4 <= len(d):
        m = d[i + 1]
        if m == marker:
            return i
        i += 2 + (d[i + 2] << 8 | d[i + 3])
    raise AssertionError(f"no marker {marker:#x}")


def rejects(d):
    with pytest.raises(ValueError):
        E.jpeg_probe(d)


@pytest.mark.parametrize("subsampling", [0, 1, 2])
@pytest.mark.parametrize("restart", [{}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1}])
def test_accepts_supported_samplings(subsampling, restart):
    d = encode(37, 53, quality=90, subsampling=subsampling, **restart)
    H, W, ws = E.jpeg_probe(d)
    assert (H, W) == (37, 53)
    assert ws > len(d)


def test_fixture_dimensions_and_workspace():
    H, W, ws = E.jpeg_probe(open(os.path.join(GOLDEN, "jpeg_depth_4.jpg"), "rb").read())
    assert (H, W) == (1200, 686)
    # coefficients (2 bytes) and pixels (1 byte) of every block of the 4:2:0 frame, MCU-padded, are a lower bound
    blocks = 43 * 75 * 4 + 2 * 43 * 75
    assert blocks * 64 * 3 < ws < blocks * 64 * 3 + 4 * 63043 + (1 << 20)
    H, W, _ = E.jpeg_probe(open(os.path.join(GOLDEN, "jpeg_dis_bag.jpg"), "rb").read())
    assert (H, W) == (3872, 2592)


def test_rejects_progressive():
    rejects(encode(32, 32, progressive=True))


def test_rejects_greyscale_and_cmyk():
    rejects(encode(32, 32, mode="L"))
    rejects(encode(32, 32, mode="CMYK"))


def test_rejects_other_samplings():
    d = bytearray(encode(32, 32, subsampling=2))
    sof = segment(d, 0xC0)
    d[sof + 4 + 7] = 0x41                                  # Y 4x1 with 1x1 chroma: 4:1:1
    rejects(bytes(d))
    d[sof + 4 + 7] = 0x12                                  # Y 1x2: 4:4:0
    rejects(bytes(d))
    d[sof + 4 + 7] = 0x22
    d[sof + 4 + 10] = 0x21                                 # chroma not 1x1
    rejects(bytes(d))


def test_rejects_lossless_sof3():
    d = bytearray(encode(32, 32))
    d[segment(d, 0xC0) + 1] = 0xC3
    rejects(bytes(d))


def test_rejects_truncated_headers():
    d = encode(32, 32)
    sos = segment(d, 0xDA)
    for n in (0, 1, 3, 20, sos - 1, sos + 5):
        rejects(d[:n])


def test_rejects_bad_table_lengths():
    d = bytearray(encode(32, 32))
    dht = segment(d, 0xC4)
    bad = bytearray(d)
    bad[dht + 2:dht + 4] = b"\xff\xff"                     # runs past the end of the file
    rejects(bytes(bad))
    bad = bytearray(d)
    bad[dht + 4 + 1 + 15] = 200                            # 16-bit code count past the segment's symbols
    rejects(bytes(bad))
    dqt = segment(d, 0xDB)
    bad = bytearray(d)
    bad[dqt + 2:dqt + 4] = b"\x00\x10"                     # a quantisation table shorter than 64 entries
    rejects(bytes(bad))


def test_rejects_missing_sos():
    d = encode(32, 32)
    sos = segment(d, 0xDA)
    rejects(d[:sos] + b"\xff\xd9")


def test_rejects_zero_sized_frame():
    for off in (5, 7):                                     # height, width
        d = bytearray(encode(32, 32))
        sof = segment(d, 0xC0)
        d[sof + off:sof + off + 2] = b"\x00\x00"
        rejects(bytes(d))


def test_rejects_adobe_rgb():
    d = encode(32, 32)
    app0 = segment(d, 0xE0)                                # without JFIF, libjpeg follows Adobe's transform
    d = d[:app0] + d[app0 + 2 + (d[app0 + 2] << 8 | d[app0 + 3]):]
    app14 = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"   # transform 0: RGB
    rejects(d[:2] + app14 + d[2:])
    E.jpeg_probe(d[:2] + app14[:-1] + b"\x01" + d[2:])                 # transform 1: YCbCr


def test_rejects_huffman_table_with_an_all_ones_code():
    """libjpeg rejects a table that uses the all-ones code of a length (Pillow raises); so does the probe."""
    d = encode(32, 32)
    i = segment(d, 0xC4)
    assert d[i + 4] == 0x00                                # the first table is the luminance DC table
    counts = list(d[i + 5:i + 21])
    k = sum(counts[:9])
    counts[8] += 1                                         # one more 9-bit code fills the code space
    seg = bytes([0x00]) + bytes(counts) + d[i + 21:i + 21 + k] + b"\x0b" + d[i + 21 + k:i + 2 + (d[i + 2] << 8 | d[i + 3])]
    bad = d[:i] + b"\xff\xc4" + (len(seg) + 2).to_bytes(2, "big") + seg + d[i + 2 + (d[i + 2] << 8 | d[i + 3]):]
    with pytest.raises(OSError):
        Image.open(io.BytesIO(bad)).convert("RGB")
    rejects(bad)
