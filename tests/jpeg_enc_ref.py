"""Numpy restatement of the baseline JPEG encoder that cv2.imencode('.jpg') runs (OpenCV 4.13 on libjpeg-turbo 3.1):
parameter resolution, headers, colour conversion, edge replication and downsampling, dummy blocks, ISLOW forward
DCT, reciprocal quantisation and Huffman coding.  `encode` returns the file and the intermediate coefficients and
per-block bit counts, so that a device mismatch can be located.  DESIGN.md §2 states the rules."""
from __future__ import annotations

import numpy as np

# ITU T.81 Annex K: K.1 base quantisation tables (natural order), K.3 standard Huffman tables (BITS, HUFFVAL)
BASE_Q = (
    np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
              14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
              49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64),
    np.array([17, 18, 24, 47] + [99] * 4 + [18, 21, 26, 66] + [99] * 4 + [24, 26, 56] + [99] * 5 + [47, 66] + [99] * 38,
             np.int64),
)
DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
DC_VALS = (list(range(12)), list(range(12)))
AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119])
_AC_TAIL = [(r << 4) | s for r in range(16) for s in range(1, 11)]


def _ac_vals(head):
    return head + [v for v in _AC_TAIL if v not in head]


AC_VALS = (
    _ac_vals([0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
              0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
              0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
              0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
              0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
              0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
              0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
              0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
              0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2]),
    _ac_vals([0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
              0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
              0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
              0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
              0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
              0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
              0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
              0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
              0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
              0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8]),
)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])     # zigzag index -> natural index
SAMPLING = {"411": (4, 1), "420": (2, 2), "422": (2, 1), "440": (1, 2), "444": (1, 1)}
CV2_SAMPLING = {"411": 0x411111, "420": 0x221111, "422": 0x211111, "440": 0x121111, "444": 0x111111}


def cv2_params(quality=95, sampling="420", restart_interval=0, luma_quality=None, chroma_quality=None):
    """The cv2.imencode parameter list that encode() with these arguments equals."""
    p = [1, int(quality), 7, CV2_SAMPLING[sampling], 4, int(restart_interval)]
    if luma_quality is not None:
        p += [5, int(luma_quality)]
    if chroma_quality is not None:
        p += [6, int(chroma_quality)]
    return p


def quality_scale(q):
    """libjpeg's jpeg_quality_scaling: 1..100, percentage scale of the base tables."""
    q = min(max(int(q), 1), 100)
    return 5000 // q if q < 50 else 200 - 2 * q


def resolve(channels, quality=95, sampling="420", restart_interval=0, luma_quality=None, chroma_quality=None):
    """-> (scale of table 0, scale of table 1, luma h, luma v, restart interval) as OpenCV sets up libjpeg.
    quality is clamped to 0..100 by OpenCV, then to 1..100 by libjpeg.  A luma quality of 0 or more replaces
    quality and, unless a chroma quality is also given, the chroma quality; a chroma quality alone is ignored.
    Unequal luma and chroma qualities turn subsampling off."""
    if sampling not in SAMPLING:
        raise ValueError(f"sampling must be one of {sorted(SAMPLING)}, got {sampling!r}")
    q = min(max(int(quality), 0), 100)
    lq = cq = -1
    if luma_quality is not None and int(luma_quality) >= 0:
        lq = min(int(luma_quality), 100)
        q = lq
        cq = lq
    if chroma_quality is not None and int(chroma_quality) >= 0 and lq >= 0:
        cq = min(int(chroma_quality), 100)
    h, v = SAMPLING[sampling]
    s0 = s1 = quality_scale(q)
    if lq >= 0:
        s0, s1 = quality_scale(lq), quality_scale(cq)
        if lq != cq:
            h, v = 1, 1
    if channels == 1:
        h, v = 1, 1
    return s0, s1, h, v, min(max(int(restart_interval), 0), 65535)


def quant_table(t, scale):
    """Natural-order baseline table: (base * scale + 50) // 100 clamped to 1..255."""
    return np.clip((BASE_Q[t] * scale + 50) // 100, 1, 255)


def huff_codes(bits, vals):
    """Annex C code assignment -> {symbol: (code, length)}."""
    codes, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            codes[vals[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return codes


DC_CODES = tuple(huff_codes(DC_BITS[t], DC_VALS[t]) for t in range(2))
AC_CODES = tuple(huff_codes(AC_BITS[t], AC_VALS[t]) for t in range(2))


def _seg(marker, payload):
    return bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + bytes(payload)


def header(h, w, channels, **kw):
    """SOI, APP0 JFIF 1.01, DQT per table, SOF0, DHT per table (DC0, AC0, DC1, AC1), DRI when restarting, SOS."""
    s0, s1, hs, vs, ri = resolve(channels, **kw)
    nt = 1 if channels == 1 else 2
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t, s in list(enumerate((s0, s1)))[:nt]:
        out += _seg(0xDB, [t] + quant_table(t, s)[ZIGZAG].tolist())
    comps = [(1, hs, vs, 0)] + ([(2, 1, 1, 1), (3, 1, 1, 1)] if channels == 3 else [])
    sof = [8, h >> 8, h & 255, w >> 8, w & 255, len(comps)]
    for cid, hh, vv, tq in comps:
        sof += [cid, hh << 4 | vv, tq]
    out += _seg(0xC0, sof)
    for t in range(nt):
        out += _seg(0xC4, [t] + DC_BITS[t] + DC_VALS[t])
        out += _seg(0xC4, [0x10 | t] + AC_BITS[t] + AC_VALS[t])
    if ri:
        out += _seg(0xDD, [ri >> 8, ri & 255])
    sos = [len(comps)]
    for cid, _, _, tq in comps:
        sos += [cid, tq << 4 | tq]
    return out + _seg(0xDA, sos + [0, 63, 0])


def rgb_to_ycc(img):
    """libjpeg's rgb_ycc_convert: 16-bit fixed point, Cb / Cr offset 128 with the ONE_HALF - 1 rounding."""
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))

    def fix(x):
        return int(x * 65536 + 0.5)
    half, off = 1 << 15, 128 << 16
    y = (fix(0.299) * r + fix(0.587) * g + fix(0.114) * b + half) >> 16
    cb = (-fix(0.16874) * r - fix(0.33126) * g + fix(0.5) * b + off + half - 1) >> 16
    cr = (fix(0.5) * r - fix(0.41869) * g - fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def geometry(h, w, channels, hs, vs):
    """Per component: (h, v, width in blocks, height in blocks); MCU columns and rows."""
    if channels == 1:
        return [(1, 1, -(-w // 8), -(-h // 8))], -(-w // 8), -(-h // 8)
    comps = [(hs, vs)] + [(1, 1)] * 2
    geo = [(ch, cv, -(-w * ch // (hs * 8)), -(-h * cv // (vs * 8))) for ch, cv in comps]
    return geo, -(-w // (hs * 8)), -(-h // (vs * 8))


def component_plane(plane, h, w, ch, cv, hs, vs, rows, cols):
    """Component samples [rows, cols] after edge replication and downsampling.  Full-resolution columns are
    replicated past the right edge; rows past the bottom replicate row h-1 within the last row group of vs rows,
    and component rows past the last group replicate the group's last component row."""
    he, ve = hs // ch, vs // cv
    cy = np.minimum(np.arange(rows), -(-h // vs) * cv - 1)
    fy = np.minimum(cy[:, None] * ve + np.arange(ve)[None, :], h - 1)          # [rows, ve]
    fx = np.minimum(np.arange(cols)[:, None] * he + np.arange(he)[None, :], w - 1)  # [cols, he]
    s = plane[fy[:, None, :, None], fx[None, :, None, :]].sum(axis=(2, 3))
    if he == 1 and ve == 1:
        return s
    if he == 2 and ve == 1:       # h2v1: bias 0, 1, 0, 1, ... across the row
        return (s + (np.arange(cols) & 1)[None, :]) >> 1
    if he == 2 and ve == 2:       # h2v2: bias 1, 2, 1, 2, ...
        return (s + 1 + (np.arange(cols) & 1)[None, :]) >> 2
    n = he * ve                   # generic integer downsampler
    return (s + n // 2) // n


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def fdct_islow(blocks):
    """jfdctint.c on int64 blocks [..., 8, 8] of samples - 128; output scaled by 8 like libjpeg's."""
    d = blocks.astype(np.int64).copy()
    for pas in range(2):
        a = d if pas == 0 else np.swapaxes(d, -1, -2).copy()
        t0, t7 = a[..., 0] + a[..., 7], a[..., 0] - a[..., 7]
        t1, t6 = a[..., 1] + a[..., 6], a[..., 1] - a[..., 6]
        t2, t5 = a[..., 2] + a[..., 5], a[..., 2] - a[..., 5]
        t3, t4 = a[..., 3] + a[..., 4], a[..., 3] - a[..., 4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        o = np.empty_like(a)
        sh = 11 if pas == 0 else 15
        if pas == 0:
            o[..., 0], o[..., 4] = (t10 + t11) << 2, (t10 - t11) << 2
        else:
            o[..., 0], o[..., 4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
        z1 = (t12 + t13) * 4433
        o[..., 2] = _descale(z1 + t13 * 6270, sh)
        o[..., 6] = _descale(z1 - t12 * 15137, sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * 9633
        t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        o[..., 7] = _descale(t4 + z1 + z3, sh)
        o[..., 5] = _descale(t5 + z2 + z4, sh)
        o[..., 3] = _descale(t6 + z2 + z3, sh)
        o[..., 1] = _descale(t7 + z1 + z4, sh)
        d = o if pas == 0 else np.swapaxes(o, -1, -2)
    return d


def reciprocal(q):
    """libjpeg-turbo's compute_reciprocal for divisor 8 * q: (multiplier, correction, shift) with
    |x| / d == ((|x| + correction) * multiplier) >> shift, rounding half away from zero."""
    d = 8 * np.asarray(q, np.int64)
    b = np.floor(np.log2(d)).astype(np.int64)
    r = 16 + b
    fq, fr = (np.int64(1) << r) // d, (np.int64(1) << r) % d
    c = d // 2
    exact = fr == 0
    fq = np.where(exact, fq >> 1, np.where(fr > d // 2, fq + 1, fq))
    c = np.where(~exact & (fr <= d // 2), c + 1, c)
    r = np.where(exact, r - 1, r)
    return fq, c, r


def quantize(coef, q):
    fq, c, r = reciprocal(q)
    a = np.abs(coef)
    v = ((a + c) * fq) >> r
    return np.where(coef < 0, -v, v)


def coefficients(img, **kw):
    """-> (coef int16 [nblocks, 64] zigzag in scan order, comp [nblocks], is_dummy [nblocks], mcu [nblocks],
    geometry).  Dummy blocks have AC zero and the quantised DC of the block before them in their MCU."""
    img = np.asarray(img)
    channels = 1 if img.ndim == 2 or img.shape[2] == 1 else 3
    h, w = img.shape[:2]
    s0, s1, hs, vs, ri = resolve(channels, **kw)
    geo, mx, my = geometry(h, w, channels, hs, vs)
    if channels == 1:
        planes = [img.reshape(h, w).astype(np.int64)]
        hs = vs = 1
    else:
        planes = list(rgb_to_ycc(img))
    per_comp = []
    for c, (ch, cv, wib, hib) in enumerate(geo):
        rows, cols = my * cv * 8, mx * ch * 8
        s = component_plane(planes[c], h, w, ch, cv, hs, vs, rows, cols) - 128
        blk = s.reshape(my * cv, 8, mx * ch, 8).transpose(0, 2, 1, 3)
        q = quant_table(0 if c == 0 else 1, s0 if c == 0 else s1)
        co = quantize(fdct_islow(blk).reshape(my * cv, mx * ch, 64), q)[..., ZIGZAG]
        per_comp.append(co)
    out, comp, dummy, mcu = [], [], [], []
    for m in range(mx * my):
        yy, xx = divmod(m, mx)
        for c, (ch, cv, wib, hib) in enumerate(geo):
            for by in range(cv):
                for bx in range(ch):
                    gy, gx = yy * cv + by, xx * ch + bx
                    if gx < wib and gy < hib:
                        out.append(per_comp[c][gy, gx].copy())
                        dummy.append(False)
                    else:
                        z = np.zeros(64, np.int64)
                        z[0] = out[-1][0]        # DC of the block before it in this MCU
                        out.append(z)
                        dummy.append(True)
                    comp.append(c)
                    mcu.append(m)
    return (np.array(out, np.int16), np.array(comp, np.int8), np.array(dummy), np.array(mcu, np.int64),
            (geo, mx, my, ri))


def _nbits(v):
    return int(abs(int(v))).bit_length()


def encode(img, **kw):
    """cv2.imencode('.jpg', img, cv2_params(**kw)) -> dict(data=bytes, header=bytes, coef, comp, dummy,
    bits=int64 [nblocks] Huffman bits of each block, segments=list of unstuffed segment bytes)."""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3)):
        raise ValueError(f"expected uint8 [H, W], [H, W, 1] or [H, W, 3], got {img.dtype} {img.shape}")
    channels = 1 if img.ndim == 2 or img.shape[2] == 1 else 3
    hdr = header(img.shape[0], img.shape[1], channels, **kw)
    coef, comp, dummy, mcu, (geo, mx, my, ri) = coefficients(img, **kw)
    nb = len(coef)
    bits = np.zeros(nb, np.int64)
    segments, acc, nacc, cur = [], bytearray(), 0, 0
    last = [0, 0, 0]
    seg_of = mcu // ri if ri else np.zeros(nb, np.int64)

    def put(code, ln):
        nonlocal cur, nacc
        cur = (cur << ln) | (code & ((1 << ln) - 1))
        nacc += ln
        while nacc >= 8:
            nacc -= 8
            acc.append((cur >> nacc) & 255)
        cur &= (1 << nacc) - 1

    def flush():
        nonlocal acc, nacc, cur
        if nacc:
            put((1 << (8 - nacc)) - 1, 8 - nacc)
        segments.append(bytes(acc))
        acc = bytearray()

    for b in range(nb):
        if b and seg_of[b] != seg_of[b - 1]:
            flush()
            last = [0, 0, 0]
        c = int(comp[b])
        t = 0 if c == 0 else 1
        blk = coef[b].astype(np.int64)
        n0 = nacc + 8 * len(acc)
        diff = int(blk[0]) - last[c]
        last[c] = int(blk[0])
        s = _nbits(diff)
        put(*DC_CODES[t][s])
        if s:
            put(diff if diff > 0 else diff - 1, s)
        run = 0
        for k in range(1, 64):
            v = int(blk[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                put(*AC_CODES[t][0xF0])
                run -= 16
            s = _nbits(v)
            put(*AC_CODES[t][(run << 4) | s])
            put(v if v > 0 else v - 1, s)
            run = 0
        if run:
            put(*AC_CODES[t][0x00])
        bits[b] = nacc + 8 * len(acc) - n0
    flush()
    body = bytearray(hdr)
    for i, seg in enumerate(segments):
        if i:
            body += bytes([0xFF, 0xD0 + (i - 1) % 8])
        body += seg.replace(b"\xff", b"\xff\x00")
    body += b"\xff\xd9"
    return dict(data=bytes(body), header=hdr, coef=coef, comp=comp, dummy=dummy, bits=bits, segments=segments)
