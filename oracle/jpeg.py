"""CPU oracle for the GPU baseline-JPEG decoder (genpercept_b200/csrc/jpeg.cu).  TEST INFRASTRUCTURE ONLY.

Plain numpy / Python restatement of what Pillow (libjpeg-turbo) computes for ``Image.open(f).convert("RGB")`` on a
sequential Huffman-coded 8-bit YCbCr JPEG, with Pillow's settings (``JDCT_ISLOW``, fancy upsampling):

* the marker parser and the streams the GPU decoder accepts (everything else raises ``Unsupported``);
* sequential Huffman decoding with the DC prediction reset at each restart interval;
* libjpeg's integer ``jpeg_idct_islow`` (13-bit constants, PASS1_BITS = 2) and its post-IDCT range-limit table;
* ``h2v1`` / ``h2v2`` fancy (triangle) upsampling over the true downsampled extents, or pixel replication when the
  downsampled width is 2 or less (libjpeg's ``jinit_upsampler`` rule), and the 16-bit fixed-point YCbCr -> RGB tables;
* ``simulate_sync``: the subsequence / self-synchronisation scheme of the GPU decoder (Weissenberger & Schmidt,
  ICPP 2018) run serially, returning its coefficients and the number of passes it needed.

PINNED (tests/test_oracle_jpeg.py): ``decode`` byte for byte against Pillow, and ``simulate_sync``'s coefficients
equal to the sequential decoder's, on seeded images of every supported sampling with and without restart markers.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])       # zigzag index -> natural index


class Unsupported(ValueError):
    """The stream is not one the GPU decoder takes (Pillow decodes it, or reports it corrupt)."""


class Corrupt(ValueError):
    """The entropy-coded data is not a clean decode (libjpeg would warn and substitute)."""


def _u16(d, i):
    if i + 2 > len(d):
        raise Unsupported("truncated header")
    return d[i] << 8 | d[i + 1]


def parse(data):
    """Marker segments up to the first SOS -> dict of the frame, tables, restart interval and entropy-data offset."""
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Unsupported("no SOI")
    i, jfif, adobe, frame, dri = 2, False, None, None, 0
    qt, dc, ac = {}, {}, {}
    while True:
        if i + 4 > len(d):
            raise Unsupported("truncated header")
        if d[i] != 0xFF:
            raise Unsupported("expected a marker")
        m = d[i + 1]
        if m == 0xFF:                                 # fill byte before a marker
            i += 1
            continue
        L = _u16(d, i + 2)
        if L < 2 or i + 2 + L > len(d):
            raise Unsupported("bad segment length")
        seg = d[i + 4:i + 2 + L]
        if m == 0xE0 and len(seg) >= 14 and seg[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and seg[:5] == b"Adobe":
            adobe = seg[11]
        elif m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                n = 64 * (2 if pq else 1)
                if pq > 1 or tq > 3 or j + 1 + n > len(seg):
                    raise Unsupported("bad DQT")
                raw = seg[j + 1:j + 1 + n]
                vals = np.frombuffer(raw, dtype=">u2" if pq else np.uint8).astype(np.int32)
                q = np.zeros(64, np.int32)
                q[ZIGZAG] = vals
                qt[tq] = q
                j += 1 + n
        elif m == 0xC4:
            j = 0
            while j < len(seg):
                if j + 17 > len(seg):
                    raise Unsupported("bad DHT")
                tc, th = seg[j] >> 4, seg[j] & 15
                counts = list(seg[j + 1:j + 17])
                n = sum(counts)
                if tc > 1 or th > 3 or n > 256 or j + 17 + n > len(seg):
                    raise Unsupported("bad DHT")
                vals = list(seg[j + 17:j + 17 + n])
                if tc == 0 and any(v > 15 for v in vals):
                    raise Unsupported("bad DC table")
                (ac if tc else dc)[th] = _huff_table(counts, vals)
                j += 17 + n
        elif m == 0xDD:
            if L != 4:
                raise Unsupported("bad DRI")
            dri = _u16(d, i + 4)
        elif m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6:
                raise Unsupported("bad SOF")
            P, H, W, nf = seg[0], seg[1] << 8 | seg[2], seg[3] << 8 | seg[4], seg[5]
            if P != 8 or nf != 3 or len(seg) != 6 + 3 * nf:
                raise Unsupported("not 8-bit, 3-component")
            if H == 0 or W == 0:
                raise Unsupported("zero-sized frame")
            comps = [dict(id=seg[6 + 3 * c], h=seg[7 + 3 * c] >> 4, v=seg[7 + 3 * c] & 15, tq=seg[8 + 3 * c])
                     for c in range(3)]
            frame = dict(H=H, W=W, comps=comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported("not a sequential Huffman frame")
        elif m == 0xDA:
            if frame is None:
                raise Unsupported("SOS before SOF")
            ns = seg[0] if seg else 0
            if ns != 3 or len(seg) != 4 + 2 * ns:
                raise Unsupported("not one interleaved scan of all components")
            for c in range(3):
                if seg[1 + 2 * c] != frame["comps"][c]["id"]:
                    raise Unsupported("scan component order")
                frame["comps"][c]["td"] = seg[2 + 2 * c] >> 4
                frame["comps"][c]["ta"] = seg[2 + 2 * c] & 15
            if seg[7] != 0 or seg[8] != 63 or seg[9] != 0:
                raise Unsupported("not a sequential scan")
            start = i + 2 + L
            break
        elif m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7:
            raise Unsupported("unexpected marker")
        i += 2 + L
    comps = frame["comps"]
    if not jfif:                                       # libjpeg's default_decompress_parms for 3 components
        if adobe is not None:
            if adobe != 1:
                raise Unsupported("Adobe transform is not YCbCr")
        elif [c["id"] for c in comps] != [1, 2, 3]:
            raise Unsupported("colour space not inferred as YCbCr")
    if (comps[1]["h"], comps[1]["v"], comps[2]["h"], comps[2]["v"]) != (1, 1, 1, 1) or \
            (comps[0]["h"], comps[0]["v"]) not in ((1, 1), (2, 1), (2, 2)):
        raise Unsupported("sampling")
    for c in comps:
        if c["tq"] not in qt or c["td"] not in dc or c["ta"] not in ac:
            raise Unsupported("missing table")
    return dict(frame, qt=qt, dc=dc, ac=ac, dri=dri, start=start)


def _huff_table(counts, vals):
    """Canonical code -> {(length, code): symbol}; raises on an over-subscribed code space (as libjpeg does)."""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            table[(length, code)] = vals[k]
            code += 1
            k += 1
        if code >= (1 << length):                      # libjpeg reserves the all-ones code of each length
            raise Unsupported("bad Huffman table")
        code <<= 1
    lens, syms = np.zeros(65536, np.int64), np.zeros(65536, np.int64)    # 16-bit peek -> (length, symbol)
    for (length, c), s in table.items():                                   # length 0 = invalid code
        lo = c << (16 - length)
        lens[lo:lo + (1 << (16 - length))] = length
        syms[lo:lo + (1 << (16 - length))] = s
    return list(zip(lens.tolist(), syms.tolist()))


def unstuff(data, start):
    """Entropy-coded bytes from `start` to the terminating marker -> (unstuffed bytes, restart-interval starts as
    offsets into them).  Only RSTn markers with the expected numbers may appear; the terminating one must be EOI."""
    d = bytes(data)
    out, rst = bytearray(), []
    i = start
    while True:
        if i >= len(d):
            raise Corrupt("no EOI")
        b = d[i]
        if b != 0xFF:
            out.append(b)
            i += 1
            continue
        if i + 1 >= len(d):
            raise Corrupt("no EOI")
        n = d[i + 1]
        if n == 0:
            out.append(0xFF)
        elif 0xD0 <= n <= 0xD7:
            if n - 0xD0 != len(rst) % 8:
                raise Corrupt("restart marker out of sequence")
            rst.append(len(out))
        elif n == 0xD9:
            return bytes(out), rst
        else:
            raise Corrupt("unexpected marker in the scan")
        i += 2


class _Bits:
    def __init__(self, u):
        bits = np.concatenate([np.unpackbits(np.frombuffer(u, np.uint8)), np.zeros(80, np.uint8)])
        w = np.lib.stride_tricks.sliding_window_view(bits, 16) @ (1 << np.arange(15, -1, -1))
        self.win = w.astype(np.int64).tolist()        # 16-bit peek at every bit position (zeros past the end)
        self.n = len(u) * 8


def _layout(hdr):
    comps = hdr["comps"]
    hm, vm = comps[0]["h"], comps[0]["v"]
    mx, my = -(-hdr["W"] // (8 * hm)), -(-hdr["H"] // (8 * vm))
    blocks = []                                        # per block of an MCU: (component, dy, dx)
    for ci, c in enumerate(comps):
        for by in range(c["v"]):
            for bx in range(c["h"]):
                blocks.append((ci, by, bx))
    return mx, my, blocks


def _step(hdr, blocks, bits, state, on_coef=None):
    """Decodes one codeword (+ its extra bits) from state (p, b, k) -> the next state; raises Corrupt on an invalid
    code or a run past coefficient 63.  on_coef(k, value) receives each decoded coefficient (k = 0: the DC diff)."""
    p, b, k = state
    if p > bits.n:
        raise Corrupt("decode past the end of the data")
    c = hdr["comps"][blocks[b][0]]
    lut = hdr["dc"][c["td"]] if k == 0 else hdr["ac"][c["ta"]]
    length, sym = lut[bits.win[p]]
    if length == 0:
        raise Corrupt("bad Huffman code")
    p += length
    if k == 0:
        v = 0
        if sym:
            v = bits.win[p] >> (16 - sym)
            p += sym
            if v < (1 << (sym - 1)):
                v -= (1 << sym) - 1
        if on_coef:
            on_coef(0, v)
        k = 1
    else:
        r, s = sym >> 4, sym & 15
        if s:
            k += r
            if k > 63:
                raise Corrupt("run past coefficient 63")
            v = bits.win[p] >> (16 - s)
            p += s
            if v < (1 << (s - 1)):
                v -= (1 << s) - 1
            if on_coef:
                on_coef(k, v)
            k += 1
        elif r == 15:
            k += 16
            if k > 64:
                raise Corrupt("run past coefficient 63")
        else:
            k = 64
    if k == 64:
        b, k = b + 1, 0
        if b == len(blocks):
            b = 0
    return p, b, k


def _intervals(hdr, u, rst):
    mx, my, blocks = _layout(hdr)
    total = mx * my
    ri = hdr["dri"] or total
    n = -(-total // ri)
    if len(rst) != n - 1:
        raise Corrupt("restart marker count")
    starts = [0] + [8 * r for r in rst]
    ends = starts[1:] + [8 * len(u)]
    return [(starts[i], ends[i], min(ri, total - i * ri)) for i in range(n)]


def _planes(hdr):
    mx, my, _ = _layout(hdr)
    return [np.zeros((my * c["v"], mx * c["h"], 64), np.int32) for c in hdr["comps"]]


def _store(hdr, planes, blocks, mcu, b, k, v):
    mx = -(-hdr["W"] // (8 * hdr["comps"][0]["h"]))
    ci, by, bx = blocks[b]
    c = hdr["comps"][ci]
    planes[ci][(mcu // mx) * c["v"] + by, (mcu % mx) * c["h"] + bx, k] = v


def decode_coefficients(hdr, u, rst):
    """Sequential decode -> per-component [bh, bw, 64] coefficients in zigzag order, DC made absolute."""
    mx, my, blocks = _layout(hdr)
    bits = _Bits(u)
    planes = _planes(hdr)
    mcu0 = 0
    for a, z, n_mcu in _intervals(hdr, u, rst):
        state, pred = (a, 0, 0), [0, 0, 0]
        for m in range(mcu0, mcu0 + n_mcu):
            for b in range(len(blocks)):
                ci = blocks[b][0]

                def put(k, v, m=m, b=b, ci=ci):
                    if k == 0:
                        pred[ci] += v
                        v = pred[ci]
                        if not -32768 <= v <= 32767:
                            raise Corrupt("DC out of range")
                    _store(hdr, planes, blocks, m, b, k, v)
                while True:
                    state = _step(hdr, blocks, bits, state, put)
                    if state[2] == 0:
                        break
                if state[0] > z:
                    raise Corrupt("interval data exhausted")
        mcu0 += n_mcu
    return planes


def simulate_sync(hdr, u, rst, sub_bits, max_passes=64):
    """The GPU decoder's scheme, serially: each restart interval is cut into subsequences of `sub_bits` bits; every
    pass decodes each subsequence from its entry state (p, b, k) to the first codeword boundary at or past its end,
    and the exit becomes the next subsequence's entry.  Interval starts are exact entries (p, 0, 0); the rest start
    as guesses (start, 0, 0), and keep their entry while the predecessor's decode hits an invalid code.  Returns
    (coefficients as decode_coefficients gives them, passes until no entry changed) or (None, max_passes) when it did
    not converge."""
    mx, my, blocks = _layout(hdr)
    bits = _Bits(u)
    subs = []                                          # (interval, start bit, end bit, head)
    ivs = _intervals(hdr, u, rst)
    for iv, (a, z, _) in enumerate(ivs):
        n = max(1, -(-(z - a) // sub_bits))
        for j in range(n):
            subs.append((iv, a + j * sub_bits, min(a + (j + 1) * sub_bits, z), j == 0))
    DEAD = None
    entry = [(s[1], 0, 0) for s in subs]

    def run(i, e, sink=None):
        _, _, end, _ = subs[i]
        st, started = e, 0
        if st is DEAD:
            return DEAD, 0
        try:
            while st[0] < end:
                if st[2] == 0:
                    started += 1
                st = _step(hdr, blocks, bits, st, sink(started) if sink else None)
        except Corrupt:
            return DEAD, started
        return st, started
    for passes in range(1, max_passes + 1):
        exits = [run(i, entry[i]) for i in range(len(subs))]
        # a predecessor that hit an invalid code keeps its successor's entry: at the fixpoint that is either garbage
        # past an interval's last block or a corrupt stream, which the writing pass reports
        new = [entry[i] if subs[i][3] or exits[i - 1][0] is DEAD else exits[i - 1][0] for i in range(len(subs))]
        if new == entry:
            break
        entry = new
    else:
        return None, max_passes
    # exclusive per-interval scan of the block counts, then the writing pass with the DC prediction per interval
    planes, base, pred, mcu0 = _planes(hdr), 0, [0, 0, 0], 0
    iv_mcu0 = np.cumsum([0] + [n for _, _, n in ivs]).tolist()
    for i, (iv, _, _, head) in enumerate(subs):
        if head:
            base, pred = 0, [0, 0, 0]
        expected = ivs[iv][2] * len(blocks)

        def sink(started, i=i, iv=iv, base=base):
            idx = base + started - 1

            def put(k, v):
                if idx >= expected:
                    return
                mcu, b = iv_mcu0[iv] + idx // len(blocks), idx % len(blocks)
                if k == 0:
                    ci = blocks[b][0]
                    pred[ci] += v
                    v = pred[ci]
                _store(hdr, planes, blocks, mcu, b, k, v)
            return put
        _, n = run(i, entry[i], sink)
        base += n
    return planes, passes


def idct_islow(coef_zz, q_natural):
    """libjpeg's jpeg_idct_islow on [N, 64] zigzag coefficients with a natural-order quantisation table -> uint8
    [N, 8, 8] (the +128 level shift and the post-IDCT range-limit table included).  Raises Corrupt when a dequantised
    coefficient or a pass-1 value leaves int16, or an output before the level shift leaves [-512, 511]: outside that
    window libjpeg-turbo's SIMD IDCT (16-bit dequantisation, saturating packs) and its C version give other bytes."""
    c = np.zeros_like(coef_zz, dtype=np.int64)
    c[:, ZIGZAG] = coef_zz
    x = (c * q_natural.astype(np.int64)).reshape(-1, 8, 8)       # [N, row v, col u]
    if x.size and (x.min() < -32768 or x.max() > 32767):
        raise Corrupt("dequantised coefficient outside int16")

    def one_d(s0, s1, s2, s3, s4, s5, s6, s7):
        z1 = (s2 + s6) * 4433
        tmp2 = z1 + s6 * -15137
        tmp3 = z1 + s2 * 6270
        tmp0 = (s0 + s4) << 13
        tmp1 = (s0 - s4) << 13
        t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        t0, t1, t2, t3 = s7, s5, s3, s1
        z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
        z5 = (z3 + z4) * 9633
        t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
        return [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    cols = one_d(*[x[:, r, :] for r in range(8)])                 # pass 1 over columns: rows of the output
    ws = np.stack([(v + (1 << 10)) >> 11 for v in cols], axis=1)  # DESCALE(, CONST_BITS - PASS1_BITS)
    if ws.size and (ws.min() < -32768 or ws.max() > 32767):
        raise Corrupt("IDCT pass-1 value outside int16")
    rows = one_d(*[ws[:, :, j] for j in range(8)])
    y = np.stack([(v + (1 << 17)) >> 18 for v in rows], axis=2)  # DESCALE(, CONST_BITS + PASS1_BITS + 3)
    if y.size and (y.min() < -512 or y.max() > 511):
        raise Corrupt("IDCT output outside [-512, 511]")
    idx = y & 1023
    out = np.where(idx < 128, idx + 128, np.where(idx < 512, 255, np.where(idx < 896, 0, idx - 896)))
    return out.astype(np.uint8)


def _plane_pixels(coefs, q):
    bh, bw, _ = coefs.shape
    px = idct_islow(coefs.reshape(-1, 64), q).reshape(bh, bw, 8, 8)
    return px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def _upsample(p, H, W, h2, v2):
    """One chroma plane at its true downsampled extent -> H x W by libjpeg's fancy filter (or replication)."""
    dh, dw = -(-H // (2 if v2 else 1)), -(-W // (2 if h2 else 1))
    if not h2:
        return p[:H, :W].astype(np.int32)
    x = p[:dh].astype(np.int32)
    if dw <= 2:                                         # jinit_upsampler: no fancy filter for narrow planes
        x = np.repeat(x[:, :dw], 2, axis=1)
        return (np.repeat(x, 2, axis=0) if v2 else x)[:H, :W]
    x = x[:, :dw]
    if v2:
        up = np.concatenate([x[:1], x[:-1]])
        dn = np.concatenate([x[1:], x[-1:]])
        rows = []
        for nb in (up, dn):
            cs = 3 * x + nb
            left = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
            right = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
            even = (3 * cs + left + 8) >> 4
            odd = (3 * cs + right + 7) >> 4
            even[:, 0] = (4 * cs[:, 0] + 8) >> 4
            odd[:, -1] = (4 * cs[:, -1] + 7) >> 4
            rows.append(np.stack([even, odd], axis=2).reshape(dh, 2 * dw))
        out = np.stack(rows, axis=1).reshape(2 * dh, 2 * dw)
    else:
        left = np.concatenate([x[:, :1], x[:, :-1]], axis=1)
        right = np.concatenate([x[:, 1:], x[:, -1:]], axis=1)
        even = (3 * x + left + 1) >> 2
        odd = (3 * x + right + 2) >> 2
        even[:, 0] = x[:, 0]
        odd[:, -1] = x[:, -1]
        out = np.stack([even, odd], axis=2).reshape(dh, 2 * dw)
    return out[:H, :W]


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert: 16-bit fixed-point tables, results through the 0..255 range limit."""
    cb, cr = cb - 128, cr - 128
    r = y + ((91881 * cr + 32768) >> 16)
    g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def pixels(hdr, planes):
    H, W = hdr["H"], hdr["W"]
    c0 = hdr["comps"][0]
    px = [_plane_pixels(planes[i], hdr["qt"][hdr["comps"][i]["tq"]]) for i in range(3)]
    y = px[0][:H, :W].astype(np.int32)
    cb = _upsample(px[1], H, W, c0["h"] == 2, c0["v"] == 2)
    cr = _upsample(px[2], H, W, c0["h"] == 2, c0["v"] == 2)
    return ycc_to_rgb(y, cb, cr)


def decode(data):
    """``np.asarray(Image.open(f).convert("RGB"))`` for a stream ``parse`` accepts -> uint8 [H, W, 3]."""
    hdr = parse(data)
    u, rst = unstuff(data, hdr["start"])
    return pixels(hdr, decode_coefficients(hdr, u, rst))
