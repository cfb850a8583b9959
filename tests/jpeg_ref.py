"""numpy restatement of the baseline JPEG decode that `decode_jpeg_batch` runs on the device, stage by stage, so a
device mismatch can be located: header parse, destuff + restart segments, Huffman decode (Python), DC prediction,
libjpeg's ISLOW integer IDCT, libjpeg-turbo's fancy chroma upsampling, its 16-bit YCbCr -> BGR tables, and the EXIF
orientation OpenCV's imread applies.  Rounding rules are libjpeg-turbo 3.1's as cv2 4.13 runs them (checked against
live cv2.imdecode by tests/test_jpeg_host.py).

The entropy decoder keeps the device's status rules, in place of libjpeg's warning and grey fill:
  BAD_MARKER  a marker other than RSTn / EOI inside the entropy-coded data (the data ends there);
  BAD_RST     an RST marker out of sequence, or more RST markers than the restart interval implies (the last segment
              ends at the first extra one);
  BAD_CODE    a code no table holds, BAD_INDEX a nonzero coefficient past k = 63: the segment's decode stops there;
  TRUNCATED   a segment whose data runs out before its last block: a codeword would start at or past the end of the
              segment's bits, the last block ends past them, or restart segments are missing.  Not set for the
              blocks after a BAD_CODE / BAD_INDEX stop."""
from __future__ import annotations

import numpy as np

# statuses (include/yolob200.h: YB_JPEG_*)
BAD_MARKER, BAD_RST, BAD_CODE, BAD_INDEX, TRUNCATED = 1, 2, 4, 8, 16

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])   # zigzag index -> natural index


class Unsupported(ValueError):
    pass


def _u16(b, o, le=False):
    return (b[o + 1] << 8 | b[o]) if le else (b[o] << 8 | b[o + 1])


def _exif_orientation(seg):
    """OpenCV's reading of an APP1 Exif block: tag 0x0112 of IFD0, SHORT; anything not in 1..8 means 1."""
    if len(seg) < 14 or seg[:6] != b"Exif\x00\x00":
        return None
    t = seg[6:]
    if t[:2] == b"II":
        le = True
    elif t[:2] == b"MM":
        le = False
    else:
        return 1
    u32 = (lambda o: int.from_bytes(t[o:o + 4], "little" if le else "big"))
    if len(t) < 8:
        return 1
    ifd = u32(4)
    if ifd + 2 > len(t):
        return 1
    cnt = _u16(t, ifd, le)
    for e in range(cnt):
        o = ifd + 2 + 12 * e
        if o + 12 > len(t):
            break
        if _u16(t, o, le) == 0x0112:
            v = _u16(t, o + 8, le)
            return v if 1 <= v <= 8 else 1
    return 1


def parse(data):
    """Header fields up to SOS.  Raises Unsupported / ValueError with the reason, as yb_jpeg_parse does."""
    b = bytes(data)
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise ValueError("not a JPEG file (no SOI)")
    p = 2
    q, dht, ri, orient, jfif, adobe = {}, {}, 0, None, False, None
    sof = None
    while True:
        while p < len(b) and b[p] != 0xFF:
            raise ValueError("marker expected")
        while p < len(b) and b[p] == 0xFF:
            p += 1
        if p >= len(b):
            raise ValueError("truncated header")
        m = b[p]
        p += 1
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7:
            continue
        if m == 0xD9:
            raise ValueError("EOI before SOS")
        if p + 2 > len(b):
            raise ValueError("truncated header")
        ln = _u16(b, p)
        if ln < 2 or p + ln > len(b):
            raise ValueError("truncated header")
        seg = b[p + 2:p + ln]
        p += ln
        if m in (0xC0, 0xC1):
            if sof is not None:
                raise ValueError("second SOF")
            if len(seg) < 6:
                raise ValueError("bad SOF")
            if seg[0] != 8:
                raise Unsupported(f"{seg[0]}-bit samples")
            H, W, nf = _u16(seg, 1), _u16(seg, 3), seg[5]
            if H == 0:
                raise Unsupported("DNL (height 0 in SOF)")
            if W == 0:
                raise ValueError("width 0")
            if nf == 4:
                raise Unsupported("4 components (CMYK / YCCK)")
            if nf not in (1, 3):
                raise Unsupported(f"{nf} components")
            if len(seg) < 6 + 3 * nf:
                raise ValueError("bad SOF")
            comps = [dict(id=seg[6 + 3 * i], h=seg[7 + 3 * i] >> 4, v=seg[7 + 3 * i] & 15, tq=seg[8 + 3 * i])
                     for i in range(nf)]
            sof = dict(H=H, W=W, comps=comps)
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise Unsupported("progressive JPEG")
        elif m in (0xC3, 0xC7, 0xCB, 0xCF):
            raise Unsupported("lossless JPEG")
        elif m in (0xC5, 0xDE):
            raise Unsupported("hierarchical JPEG")
        elif m in (0xC9, 0xCC, 0xCD):
            raise Unsupported("arithmetic coding")
        elif m == 0xC4:
            o = 0
            while o < len(seg):
                tc, th = seg[o] >> 4, seg[o] & 15
                if tc > 1 or th > 3 or o + 17 > len(seg):
                    raise ValueError("bad DHT")
                bits = list(seg[o + 1:o + 17])
                nv = sum(bits)
                if nv > 256 or o + 17 + nv > len(seg):
                    raise ValueError("bad DHT")
                dht[(tc, th)] = (bits, list(seg[o + 17:o + 17 + nv]))
                o += 17 + nv
        elif m == 0xDB:
            o = 0
            while o < len(seg):
                pq, tq = seg[o] >> 4, seg[o] & 15
                if pq > 1 or tq > 3 or o + 1 + 64 * (pq + 1) > len(seg):
                    raise ValueError("bad DQT")
                if pq == 0:
                    v = np.frombuffer(seg, np.uint8, 64, o + 1).astype(np.int32)
                else:
                    v = np.frombuffer(seg, ">u2", 64, o + 1).astype(np.int32)
                t = np.zeros(64, np.int32)
                t[ZIGZAG] = v
                q[tq] = t
                o += 1 + 64 * (pq + 1)
        elif m == 0xDD:
            if len(seg) < 2:
                raise ValueError("bad DRI")
            ri = _u16(seg, 0)
        elif m == 0xE0:
            if seg[:5] == b"JFIF\x00":
                jfif = True
        elif m == 0xE1:
            if orient is None:
                orient = _exif_orientation(seg)
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif m == 0xDA:
            if sof is None:
                raise ValueError("SOS before SOF")
            ns = seg[0] if seg else 0
            comps = sof["comps"]
            if ns != len(comps):
                raise Unsupported("several scans (non-interleaved)")
            if len(seg) < 4 + 2 * ns:
                raise ValueError("bad SOS")
            for i in range(ns):
                cid, t = seg[1 + 2 * i], seg[2 + 2 * i]
                idx = [j for j, c in enumerate(comps) if c["id"] == cid]
                if len(idx) != 1:
                    raise ValueError("SOS names an unknown component")
                if idx[0] != i:
                    raise Unsupported("SOS lists the components in another order than SOF")
                comps[idx[0]]["td"], comps[idx[0]]["ta"] = t >> 4, t & 15
            ss, se, a = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or a != 0:
                raise Unsupported("spectral selection / successive approximation")
            break
        # every other marker (APPn, COM, ...) is skipped
    nf = len(sof["comps"])
    if nf == 3:
        if adobe == 0:
            raise Unsupported("RGB JPEG (Adobe transform 0)")
        if adobe is None and not jfif and [c["id"] for c in sof["comps"]] == [82, 71, 66]:
            raise Unsupported("RGB JPEG (component ids R, G, B)")
        hv = (sof["comps"][0]["h"], sof["comps"][0]["v"])
        if hv not in ((1, 1), (2, 1), (1, 2), (2, 2)) or any((c["h"], c["v"]) != (1, 1) for c in sof["comps"][1:]):
            raise Unsupported("sampling factors " + ",".join(f"{c['h']}x{c['v']}" for c in sof["comps"]))
    else:
        if not (1 <= sof["comps"][0]["h"] <= 4 and 1 <= sof["comps"][0]["v"] <= 4):
            raise ValueError("bad sampling factors")
    for c in sof["comps"]:
        if c["tq"] not in q:
            raise ValueError(f"quantisation table {c['tq']} missing")
        for key in ((0, c["td"]), (1, c["ta"])):
            if key not in dht:
                raise ValueError(f"Huffman table {key} missing")
    o = orient or 1
    H, W = sof["H"], sof["W"]
    return dict(H=H, W=W, comps=sof["comps"], q=q, dht=dht, ri=ri, orientation=o,
                out_h=W if o >= 5 else H, out_w=H if o >= 5 else W, scan_start=p, data=b)


def _geometry(info):
    comps = info["comps"]
    H, W = info["H"], info["W"]
    if len(comps) == 1:
        bw, bh = -(-W // 8), -(-H // 8)
        return dict(mcus_x=bw, mcus_y=bh, bpm=1, blocks=[(0, 0, 0)], planes=[(bh, bw)], hmax=1, vmax=1,
                    dims=[(H, W)])
    hmax, vmax = max(c["h"] for c in comps), max(c["v"] for c in comps)
    mx, my = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    blocks = [(ci, by, bx) for ci, c in enumerate(comps) for by in range(c["v"]) for bx in range(c["h"])]
    return dict(mcus_x=mx, mcus_y=my, bpm=len(blocks), blocks=blocks, hmax=hmax, vmax=vmax,
                planes=[(my * c["v"], mx * c["h"]) for c in comps],
                dims=[(-(-H * c["v"] // vmax), -(-W * c["h"] // hmax)) for c in comps])


def _huff_lookup(bits, vals):
    """(code length, code) -> symbol, canonical assignment."""
    tab, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            tab[(ln, code)] = vals[k]
            k += 1
            code += 1
        code <<= 1
    return tab


def segments(info):
    """Destuff the entropy data and split it at RST markers -> (list of segment byte strings, status)."""
    b, p = info["data"], info["scan_start"]
    segs, cur, status, nrst = [], bytearray(), 0, 0
    n = len(b)
    while p < n:
        c = b[p]
        if c != 0xFF:
            cur.append(c)
            p += 1
            continue
        nxt = b[p + 1] if p + 1 < n else None
        if nxt is None:
            p += 1
        elif nxt == 0x00:
            cur.append(0xFF)
            p += 2
        elif nxt == 0xFF:
            p += 1
        elif 0xD0 <= nxt <= 0xD7:
            if nxt != 0xD0 + (nrst & 7):
                status |= BAD_RST
            nrst += 1
            segs.append(bytes(cur))
            cur = bytearray()
            p += 2
        elif nxt == 0xD9:
            break
        else:
            status |= BAD_MARKER
            break
    segs.append(bytes(cur))
    return segs, status


def coefficients(info):
    """-> (per component int32 [bh, bw, 64] quantised coefficients in natural order, DC prediction applied, status)."""
    g = _geometry(info)
    comps = info["comps"]
    tabs = {k: _huff_lookup(*v) for k, v in info["dht"].items()}
    coef = [np.zeros((bh, bw, 64), np.int32) for bh, bw in g["planes"]]
    total = g["mcus_x"] * g["mcus_y"]
    ri = info["ri"] or total
    nseg = -(-total // ri)
    segs, status = segments(info)
    if len(segs) > nseg:
        status |= BAD_RST
    if len(segs) < nseg:
        status |= TRUNCATED
    for s in range(min(nseg, len(segs))):
        data = segs[s]
        bits = np.unpackbits(np.frombuffer(data, np.uint8)) if data else np.zeros(0, np.uint8)
        nb = len(bits)
        pos = 0
        pred = [0] * len(comps)

        def get(n):
            nonlocal pos
            v = 0
            for i in range(n):
                v = (v << 1) | (int(bits[pos + i]) if pos + i < nb else 0)
            pos += n
            return v

        def sym(tab):
            nonlocal pos
            if pos >= nb:
                return -1           # no data left for another codeword
            code = 0
            for ln in range(1, 17):
                code = (code << 1) | (int(bits[pos + ln - 1]) if pos + ln - 1 < nb else 0)
                if (ln, code) in tab:
                    pos += ln
                    return tab[(ln, code)]
            return None

        def ext(v, s):
            return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v

        m0, m1 = s * ri, min(total, (s + 1) * ri)
        bad = False
        for m in range(m0, m1):
            my, mx = divmod(m, g["mcus_x"])
            for ci, oy, ox in g["blocks"]:
                c = comps[ci]
                if len(comps) == 1:
                    by, bx = my, mx
                else:
                    by, bx = my * c["v"] + oy, mx * c["h"] + ox
                blk = np.zeros(64, np.int32)
                t = sym(tabs[(0, c["td"])])
                if t == -1:
                    status |= TRUNCATED
                    bad = True
                    break
                if t is None:
                    status |= BAD_CODE
                    bad = True
                    break
                d = ext(get(t), t) if t else 0
                pred[ci] += d
                blk[0] = pred[ci]
                k = 1
                while k < 64:
                    rs = sym(tabs[(1, c["ta"])])
                    if rs == -1:
                        status |= TRUNCATED
                        bad = True
                        break
                    if rs is None:
                        status |= BAD_CODE
                        bad = True
                        break
                    r, sz = rs >> 4, rs & 15
                    if sz:
                        k += r
                        if k > 63:
                            status |= BAD_INDEX
                            bad = True
                            break
                        blk[ZIGZAG[k]] = ext(get(sz), sz)
                        k += 1
                    elif r == 15:
                        k += 16
                    else:
                        break
                if bad:
                    break
                if pos > nb:
                    status |= TRUNCATED
                coef[ci][by, bx] = blk
            if bad:
                break
    return coef, status


# ---- ISLOW IDCT (jidctint.c), vectorised over blocks ----
_F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(v, shift):
    """v: int64 [..., 8] -> int64 [..., 8], one Loeffler-Ligtenberg-Moschytz pass with DESCALE(shift)."""
    F = _F
    z2, z3 = v[..., 2], v[..., 6]
    z1 = (z2 + z3) * F["f0541"]
    tmp2 = z1 + z3 * -F["f1847"]
    tmp3 = z1 + z2 * F["f0765"]
    tmp0 = (v[..., 0] + v[..., 4]) << 13
    tmp1 = (v[..., 0] - v[..., 4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * F["f1175"]
    a0, a1, a2, a3 = a0 * F["f0298"], a1 * F["f2053"], a2 * F["f3072"], a3 * F["f1501"]
    z1, z2, z3, z4 = z1 * -F["f0899"], z2 * -F["f2562"], z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
    a0 += z1 + z3
    a1 += z2 + z4
    a2 += z2 + z3
    a3 += z1 + z4
    r = 1 << (shift - 1)
    out = [t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3]
    return np.stack([(o + r) >> shift for o in out], -1)


def idct_blocks(coef, qt):
    """int32 [..., 64] natural-order coefficients and int32 [64] table -> uint8 [..., 8, 8] samples."""
    d = (coef.astype(np.int64) * qt.astype(np.int64)).reshape(coef.shape[:-1] + (8, 8))
    ws = np.swapaxes(_idct_1d(np.swapaxes(d, -1, -2), 11), -1, -2)       # columns, CONST_BITS - PASS1_BITS
    out = _idct_1d(ws, 18)                                                # rows, CONST_BITS + PASS1_BITS + 3
    return (np.clip(out, -128, 127) + 128).astype(np.uint8)               # SIMD ISLOW saturates


def planes(info, coef):
    """-> per component uint8 [bh * 8, bw * 8] sample planes (MCU-padded)."""
    out = []
    for c, cf in zip(info["comps"], coef):
        bh, bw = cf.shape[:2]
        s = idct_blocks(cf, info["q"][c["tq"]])
        out.append(s.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    return out


def upsample(info, pl):
    """-> per component uint8 [H, W] planes at full resolution (libjpeg-turbo fancy upsampling)."""
    g = _geometry(info)
    H, W = info["H"], info["W"]
    res = []
    for ci, (c, p) in enumerate(zip(info["comps"], pl)):
        dh, dw = g["dims"][ci]
        a = p[:dh, :dw].astype(np.int32)
        hr, vr = g["hmax"] // c["h"], g["vmax"] // c["v"]
        if len(info["comps"]) == 1 or (hr, vr) == (1, 1):
            u = a
        elif (hr, vr) == (1, 2):
            up = np.concatenate([a[:1], a[:-1]], 0)
            dn = np.concatenate([a[1:], a[-1:]], 0)
            u = np.empty((2 * dh, dw), np.int32)
            u[0::2] = (3 * a + up + 1) >> 2
            u[1::2] = (3 * a + dn + 2) >> 2
        elif (hr, vr) == (2, 1):
            if dw > 2:
                lf = np.concatenate([a[:, :1], a[:, :-1]], 1)
                rt = np.concatenate([a[:, 1:], a[:, -1:]], 1)
                u = np.empty((dh, 2 * dw), np.int32)
                u[:, 0::2] = (3 * a + lf + 1) >> 2
                u[:, 1::2] = (3 * a + rt + 2) >> 2
                u[:, 0], u[:, -1] = a[:, 0], a[:, -1]
            else:
                u = np.repeat(a, 2, 1)
        else:   # (2, 2)
            if dw > 2:
                up = np.concatenate([a[:1], a[:-1]], 0)
                dn = np.concatenate([a[1:], a[-1:]], 0)
                u = np.empty((2 * dh, 2 * dw), np.int32)
                for r, nb in ((0, up), (1, dn)):
                    cs = 3 * a + nb
                    lf = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
                    rt = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
                    u[r::2, 0::2] = (3 * cs + lf + 8) >> 4
                    u[r::2, 1::2] = (3 * cs + rt + 7) >> 4
                    u[r::2, 0] = (4 * cs[:, 0] + 8) >> 4
                    u[r::2, -1] = (4 * cs[:, -1] + 7) >> 4
            else:
                u = np.repeat(np.repeat(a, 2, 0), 2, 1)
        res.append(u[:H, :W].astype(np.uint8))
    return res


def to_bgr(up):
    """YCbCr planes -> uint8 [H, W, 3] BGR with libjpeg's tables (jdcolor.c); one plane -> replicated grey."""
    if len(up) == 1:
        return np.repeat(up[0][:, :, None], 3, 2)
    y, cb, cr = (p.astype(np.int64) for p in up)
    x_cb, x_cr = cb - 128, cr - 128
    half = 1 << 15
    r = y + ((91881 * x_cr + half) >> 16)
    gg = y + ((-22554 * x_cb + half - 46802 * x_cr) >> 16)
    b = y + ((116130 * x_cb + half) >> 16)
    return np.clip(np.stack([b, gg, r], -1), 0, 255).astype(np.uint8)


def orient(img, o):
    """EXIF orientation as OpenCV applies it after decoding."""
    if o == 2:
        return img[:, ::-1]
    if o == 3:
        return img[::-1, ::-1]
    if o == 4:
        return img[::-1]
    if o == 5:
        return img.transpose(1, 0, 2)
    if o == 6:
        return np.rot90(img, -1)
    if o == 7:
        return img.transpose(1, 0, 2)[::-1, ::-1]
    if o == 8:
        return np.rot90(img, 1)
    return img


def decode(data, stages=False):
    """JPEG bytes -> (uint8 [H, W, 3] BGR as cv2.imread returns it, status); with stages=True a dict of every stage."""
    info = parse(data)
    coef, status = coefficients(info)
    pl = planes(info, coef)
    up = upsample(info, pl)
    bgr = to_bgr(up)
    out = np.ascontiguousarray(orient(bgr, info["orientation"]))
    if stages:
        return dict(info=info, coef=coef, planes=pl, upsampled=up, bgr=bgr, out=out, status=status)
    return out, status
