"""Pins oracle/jpeg.py byte for byte against Pillow: the sequential decoder (parser, Huffman, ISLOW IDCT, fancy
upsampling, colour), and the GPU decoder's subsequence / self-synchronisation scheme against the sequential decode."""
import io
import os

import numpy as np
import pytest
from PIL import Image

from oracle import jpeg as J

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RESTARTS = [{}, {"restart_marker_blocks": 1}, {"restart_marker_blocks": 7}, {"restart_marker_rows": 1}]


def encode(h, w, q, subsampling, seed, kind="photo", **kw):
    g = np.random.default_rng(seed)
    if kind == "noise":                                   # long codes, many 0xFF bytes, clamped pixels
        a = g.integers(0, 256, (h, w, 3)).astype(np.float64)
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        a = np.stack([np.sin(xx / 7.0 + c) * np.cos(yy / 11.0 - c) for c in range(3)], -1) * 100 + 128
        if kind == "photo":
            a = a + g.normal(0, 20, a.shape)
    buf = io.BytesIO()
    Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(buf, "JPEG", quality=q, subsampling=subsampling, **kw)
    return buf.getvalue()


def pillow(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.mark.parametrize("subsampling", [0, 1, 2])
@pytest.mark.parametrize("q", [50, 90, 100])
@pytest.mark.parametrize("size", [(1, 1), (2, 3), (7, 9), (17, 33)])
def test_decode_matches_pillow(subsampling, q, size):
    for i, kw in enumerate(RESTARTS):
        for kind in ("photo", "noise", "gradient"):
            d = encode(*size, q, subsampling, seed=size[0] * 31 + q + i, kind=kind, **kw)
            np.testing.assert_array_equal(J.decode(d), pillow(d), err_msg=f"{kw} {kind}")


@pytest.mark.parametrize("subsampling", [0, 1, 2])
def test_decode_686x1200_matches_pillow(subsampling):
    d = encode(1200, 686, 90, subsampling, seed=subsampling, restart_marker_rows=1)
    np.testing.assert_array_equal(J.decode(d), pillow(d))


def test_decode_fixture_matches_pillow():
    d = open(os.path.join(GOLDEN, "jpeg_depth_4.jpg"), "rb").read()
    np.testing.assert_array_equal(J.decode(d), pillow(d))


@pytest.mark.parametrize("subsampling", [0, 1, 2])
@pytest.mark.parametrize("restart", [{}, {"restart_marker_blocks": 7}])
@pytest.mark.parametrize("kind", ["photo", "noise"])
def test_sync_simulation_matches_sequential(subsampling, restart, kind):
    d = encode(64, 96, 90, subsampling, seed=7, kind=kind, **restart)
    hdr = J.parse(d)
    u, rst = J.unstuff(d, hdr["start"])
    ref = J.decode_coefficients(hdr, u, rst)
    for sub_bits in (512, 4096):
        got, passes = J.simulate_sync(hdr, u, rst, sub_bits, max_passes=1024)
        assert got is not None, f"no convergence at {sub_bits} bits"
        for a, b in zip(got, ref):
            np.testing.assert_array_equal(a, b)


def test_sync_passes_on_fixture():
    """The GPU decoder's subsequence length (4096 bits) converges in a few passes on a real photo."""
    d = open(os.path.join(GOLDEN, "jpeg_depth_4.jpg"), "rb").read()
    hdr = J.parse(d)
    u, rst = J.unstuff(d, hdr["start"])
    got, passes = J.simulate_sync(hdr, u, rst, 4096)
    assert got is not None and passes <= 4, passes
    for a, b in zip(got, J.decode_coefficients(hdr, u, rst)):
        np.testing.assert_array_equal(a, b)


def with_dqt(data, value):
    """`data` with every quantisation table entry rewritten to `value` (a well-formed file)."""
    d = bytearray(data)
    i = 2
    while d[i + 1] != 0xDA:
        L = d[i + 2] << 8 | d[i + 3]
        if d[i + 1] == 0xDB:
            j = i + 4
            while j < i + 2 + L:
                n = 128 if d[j] >> 4 else 64
                d[j + 1:j + 1 + n] = bytes([0, value] * 64 if n == 128 else [value] * 64)
                j += 1 + n
        i += 2 + L
    return bytes(d)


def flipped(data, offset, bit):
    """`data` with one bit of its entropy-coded segment flipped (`offset` counts from the segment's first byte)."""
    d = bytearray(data)
    d[J.parse(data)["start"] + offset] ^= 1 << bit
    return bytes(d)


# single-bit flips of this photo that decode cleanly but push IDCT values out of the window where libjpeg-turbo's C and
# SIMD IDCTs agree (a DC difference that shifts every later block)
FLIP_PHOTO = dict(h=240, w=320, q=90, subsampling=2, seed=3)
OUT_OF_WINDOW_FLIPS = [(30831, 3), (9180, 7), (28474, 2)]


def test_out_of_window_idct_is_rejected():
    """Streams Pillow decodes but whose IDCT values leave the window are Corrupt, so the pipeline takes Pillow's path."""
    d = with_dqt(encode(64, 64, 100, 0, seed=1, kind="noise"), 8)
    pillow(d)                                             # Pillow decodes it
    with pytest.raises(J.Corrupt, match="IDCT|dequantised"):
        J.decode(d)
    base = encode(**FLIP_PHOTO)
    for off, bit in OUT_OF_WINDOW_FLIPS:
        with pytest.raises(J.Corrupt, match="IDCT|dequantised"):
            J.decode(flipped(base, off, bit))


def test_bit_flips_match_pillow_or_are_rejected():
    base = encode(**FLIP_PHOTO)
    n = len(base) - J.parse(base)["start"] - 2
    g = np.random.default_rng(0)
    accepted = 0
    for _ in range(60):
        d = flipped(base, int(g.integers(0, n)), int(g.integers(0, 8)))
        try:
            got = J.decode(d)
        except ValueError:
            continue
        accepted += 1
        np.testing.assert_array_equal(got, pillow(d))
    assert accepted > 10


def test_all_ones_huffman_code_is_rejected():
    with pytest.raises(J.Unsupported, match="Huffman"):
        J._huff_table([2] + [0] * 15, [0, 1])            # codes 0 and 1 of length 1: the all-ones code is used
    J._huff_table([1, 1] + [0] * 14, [0, 1])             # codes 0 and 10
