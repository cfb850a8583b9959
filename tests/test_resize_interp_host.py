"""CPU tests of the training resize (INTER_CUBIC, INTER_AREA, INTER_LANCZOS4): the numpy restatement
(tests/resize_interp_ref.py) equals the reference-generated goldens (tests/golden/make_golden_resize_interp.py) and
live cv2.resize over random shapes; yb_resize_tables builds the restatement's tables entry for entry; the new entry
points reject bad arguments before any device work."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from tests import resize_interp_cases as K
from tests import resize_interp_ref as M
from tests import resize_ref as R


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "resize_interp.npz"))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_case_sources_are_the_goldens_sources(golden_dir):
    g = _golden(golden_dir)
    assert [tuple(c) for c in g["cases"].tolist()] == [c for _, c, _ in K.cases()]
    assert [_sha(K.source(i, c[:2])) for i, c, _ in K.cases()] == g["src_sha256"].tolist()


def test_restatement_matches_reference_goldens(golden_dir):
    g = _golden(golden_dir)
    sha = dict(zip(g["keys"].tolist(), g["sha256"].tolist()))
    checked = 0
    for i, (sh, sw, nw, nh), full in K.cases():
        img = K.source(i, (sh, sw))
        gt = K.boxes(i, sh, sw)
        for interp in K.INTERPS:
            for lb in (True, False):
                key = f"{'lb' if lb else 'st'}{interp}_{i}"
                got = M.resize_image(img, nw, nh, interp, lb)
                assert _sha(got) == sha[key], key                          # IPP off for cubic: exact
                if full:
                    assert np.array_equal(got, g[key]), key
                    assert np.array_equal(R.resize_boxes(gt, sh, sw, nw, nh, lb), g[f"box_{key}"]), key
                    if interp == 2:                                        # default cv2 (IPP on): within 1
                        d = np.abs(got.astype(np.int16) - g[f"ipp_{key}"].astype(np.int16))
                        assert d.max() <= 1, key
                checked += 1
    assert checked == len(K.cases()) * 6


def test_goldens_cover_every_area_path_and_the_copy(golden_dir):
    modes = {M.area_mode(nh, nw, sh, sw) for _, (sh, sw, nw, nh), _ in K.cases()}
    assert modes == {"fast", "float", "linear"}
    assert any((sh, sw) == (nh, nw) for _, (sh, sw, nw, nh), _ in K.cases())
    assert {nw for _, (_, _, nw, nh), full in K.cases() if not full and nw == nh} >= set(range(320, 609, 32))


def _shapes(rng, count):
    out = []
    for k in range(count):
        kind = k % 5
        if kind == 0:                                   # integer shrinks (area fast) and same size
            f = rng.integers(1, 5, 2)
            nh, nw = rng.integers(1, 80, 2)
            out.append((int(nh * f[0]), int(nw * f[1]), int(nw), int(nh)))
        elif kind == 1:                                 # tiny and thin
            out.append(tuple(int(v) for v in rng.integers(1, 12, 4)))
        else:
            out.append(tuple(int(v) for v in np.concatenate([rng.integers(1, 700, 2), rng.integers(1, 640, 2)])))
    return out


@pytest.mark.parametrize("interp", [2, 3, 4])
def test_restatement_matches_live_cv2(interp):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(31 + interp)
    worst = 0
    for sh, sw, nw, nh in _shapes(rng, 100):
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        got = M.cv2_resize(img, nw, nh, interp)
        prev = cv2.ipp.useIPP()
        try:
            cv2.ipp.setUseIPP(False)
            exact = cv2.resize(img, (nw, nh), interpolation=interp)
            cv2.ipp.setUseIPP(True)
            default = cv2.resize(img, (nw, nh), interpolation=interp)
        finally:
            cv2.ipp.setUseIPP(prev)
        assert np.array_equal(got, exact), (sh, sw, nw, nh, interp)
        worst = max(worst, int(np.abs(got.astype(np.int16) - default.astype(np.int16)).max()))
    assert worst <= (1 if interp == 2 else 0)


# ---- the C tables ------------------------------------------------------------------------------------------------

HDR = np.dtype([("interp", "<i4"), ("mode", "<i4"), ("src_h", "<i4"), ("src_w", "<i4"), ("rh", "<i4"), ("rw", "<i4"),
                ("kx", "<i4"), ("ky", "<i4"), ("x_off", "<i8"), ("y_off", "<i8"), ("xt_off", "<i8"), ("yt_off", "<i8")])
GEN = np.dtype([("s", "<i4"), ("c", "<i2", 8)])
SPAN = np.dtype([("start", "<i4"), ("count", "<i4")])
TAP = np.dtype([("s", "<i4"), ("a", "<f4")])


@pytest.fixture(scope="module")
def lib():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _tables(lib, shapes, nw, nh, letterbox, interp):
    desc = np.zeros((len(shapes), 4), np.int64)
    off = 0
    for i, (h, w) in enumerate(shapes):
        desc[i] = (off, h, w, 3 * w)
        off += 3 * h * w
    it = np.ascontiguousarray(interp, np.int32)
    nbytes = C.c_size_t()
    args = (desc.ctypes.data_as(C.c_void_p), len(shapes), nh, nw, int(letterbox), it.ctypes.data_as(C.c_void_p))
    lib.check(lib.lib.yb_resize_tables_bytes(*args, C.byref(nbytes)))
    buf = np.zeros(nbytes.value // 16 + 1, np.dtype((np.void, 16)))         # 16-byte aligned storage
    raw = buf.view(np.uint8)[: nbytes.value]
    lib.check(lib.lib.yb_resize_tables(*args, raw.ctypes.data_as(C.c_void_p), nbytes.value))
    return raw


def _check_image_tables(raw, hdr, interp, sh, sw, rh, rw):
    assert (hdr["interp"], hdr["src_h"], hdr["src_w"], hdr["rh"], hdr["rw"]) == (interp, sh, sw, rh, rw)
    if interp in (0, 1):
        assert hdr["mode"] == interp
        return
    if (sh, sw) == (rh, rw):
        assert hdr["mode"] == 5
        return
    if interp in (2, 4):
        assert hdr["mode"] == interp
        for off, dst, src in ((hdr["x_off"], rw, sw), (hdr["y_off"], rh, sh)):
            t = np.frombuffer(raw, GEN, dst, int(off))
            taps, coefs = M.generic_table(dst, src, interp)
            k = taps.shape[1]
            assert np.array_equal(np.clip(t["s"][:, None] + np.arange(k), 0, src - 1), taps)
            assert np.array_equal(t["c"][:, :k], coefs) and not t["c"][:, k:].any()
        return
    mode = M.area_mode(rh, rw, sh, sw)
    if mode == "fast":
        assert (hdr["mode"], hdr["kx"], hdr["ky"]) == (6, sw // rw, sh // rh)
    elif mode == "linear":
        assert hdr["mode"] == 8
        for off, dst, src, clamp in ((hdr["x_off"], rw, sw, True), (hdr["y_off"], rh, sh, False)):
            t = np.frombuffer(raw, GEN, dst, int(off))
            s0, s1, c0, c1 = M.area_linear_table(dst, src, clamp)
            assert np.array_equal(np.clip(t["s"], 0, src - 1), s0)
            assert np.array_equal(np.clip(t["s"] + 1, 0, src - 1), s1)
            assert np.array_equal(t["c"][:, 0], c0) and np.array_equal(t["c"][:, 1], c1)
    else:
        assert hdr["mode"] == 7
        for so, to, dst, src in ((hdr["x_off"], hdr["xt_off"], rw, sw), (hdr["y_off"], hdr["yt_off"], rh, sh)):
            spans = np.frombuffer(raw, SPAN, dst, int(so))
            want = M.area_table(dst, src)
            taps = np.frombuffer(raw, TAP, len(want), int(to))
            got = [(d, int(taps["s"][k]), taps["a"][k]) for d, (st, cnt) in enumerate(spans.tolist())
                   for k in range(st, st + cnt)]
            assert [(d, s) for d, s, _ in got] == [(d, s) for d, s, _ in want]
            assert np.array_equal(np.array([a for *_, a in got], np.float32), np.array([a for *_, a in want], np.float32))


@pytest.mark.parametrize("letterbox", [True, False])
def test_c_tables_equal_the_restatement(lib, letterbox):
    rng = np.random.default_rng(5 + letterbox)
    shapes = [(sh, sw) for sh, sw, _, _ in _shapes(rng, 60)] + [(1, 1), (1, 9), (9, 1), (64, 64), (1517, 2013)]
    for nw, nh in ((64, 48), (320, 320), (37, 91), (608, 608)):
        interp = rng.integers(0, 5, len(shapes))
        raw = _tables(lib, shapes, nw, nh, letterbox, interp)
        hdrs = np.frombuffer(raw, HDR, len(shapes))
        for (sh, sw), it, hdr in zip(shapes, interp.tolist(), hdrs):
            if letterbox:
                _, rw, rh, _, _ = R.letterbox_geometry(sh, sw, nw, nh)
            else:
                rw, rh = nw, nh
            if rw == 0 or rh == 0:
                continue
            _check_image_tables(raw, hdr, it, sh, sw, rh, rw)


def test_table_size_at_batch_64_608(lib):
    shapes = [(375, 500)] * 64
    for interp, per_image in ((2, 24320), (4, 24320)):
        raw = _tables(lib, shapes, 608, 608, False, [interp] * 64)
        assert len(raw) == 64 * 64 + 64 * per_image                       # headers + 1216 taps of 20 bytes


def _interp_rc(lib, desc, interp, n=None, new_h=32, new_w=32, letterbox=1, nbytes=1 << 20, th=True, td=True,
               tbytes=None):
    desc = np.ascontiguousarray(desc, np.int64)
    it = np.ascontiguousarray(interp, np.int32)
    fake = C.c_void_p(1 << 20)                      # never dereferenced: validation precedes any device work
    n = len(desc) if n is None else n
    args = (desc.ctypes.data_as(C.c_void_p), n, new_h, new_w, letterbox, it.ctypes.data_as(C.c_void_p))
    need = C.c_size_t()
    rc_bytes = lib.lib.yb_resize_tables_bytes(*args, C.byref(need))
    host = np.zeros(max(need.value, 64) // 16 + 1, np.dtype((np.void, 16))).view(np.uint8)
    if rc_bytes == 0:
        assert lib.lib.yb_resize_tables(*args, host.ctypes.data_as(C.c_void_p), need.value) == 0
    rc = lib.lib.yb_resize_batch_interp(fake, nbytes, desc.ctypes.data_as(C.c_void_p), fake, n, new_h, new_w, letterbox,
                                        it.ctypes.data_as(C.c_void_p), host.ctypes.data_as(C.c_void_p) if th else None,
                                        fake if td else None, need.value if tbytes is None else tbytes, fake, None,
                                        None)
    return rc_bytes, rc


def test_new_entry_points_reject_bad_arguments(lib):
    ok = [[0, 10, 20, 60]]
    for bad in (-1, 5, 6):
        assert _interp_rc(lib, ok, [bad]) == (-1, -1)
    assert b"interp" in lib.lib.yb_last_error_string()
    assert _interp_rc(lib, [[0, 0, 20, 60]], [2]) == (-1, -1)                 # zero-sized image
    assert _interp_rc(lib, [[0, 1, 1000, 3000]], [3]) == (-1, -1)             # letterbox to an empty resize
    assert b"empty" in lib.lib.yb_last_error_string()
    assert _interp_rc(lib, ok, [2], letterbox=2) == (-1, -1)
    assert _interp_rc(lib, ok, [2], new_w=0) == (-1, -1)
    assert _interp_rc(lib, ok, [2], n=0) == (-1, -1)
    assert _interp_rc(lib, [[0, 10, 20, 59]], [2])[1] == -1                   # pitch < 3 * w
    assert _interp_rc(lib, [[64, 10, 20, 60]], [4], nbytes=600)[1] == -1      # past the end of the buffer
    assert _interp_rc(lib, ok, [4], th=False) == (0, -1)                      # the two table copies go together
    assert _interp_rc(lib, ok, [4], td=False) == (0, -1)
    assert b"both" in lib.lib.yb_last_error_string()
    assert _interp_rc(lib, ok, [4], tbytes=64) == (0, -1)                     # wrong table size
    # the table size must be exact, and the buffer aligned
    desc = np.ascontiguousarray(ok, np.int64)
    it = np.array([2], np.int32)
    args = (desc.ctypes.data_as(C.c_void_p), 1, 32, 32, 1, it.ctypes.data_as(C.c_void_p))
    need = C.c_size_t()
    assert lib.lib.yb_resize_tables_bytes(*args, C.byref(need)) == 0
    buf = np.zeros(need.value // 16 + 2, np.dtype((np.void, 16))).view(np.uint8)
    assert lib.lib.yb_resize_tables(*args, buf.ctypes.data_as(C.c_void_p), need.value - 1) == -1
    assert lib.lib.yb_resize_tables(*args, buf[4:].ctypes.data_as(C.c_void_p), need.value) == -1
    assert lib.lib.yb_resize_tables_bytes(*args, None) == -1


def test_tables_built_for_another_call_are_rejected(lib):
    desc = np.ascontiguousarray([[0, 10, 20, 60], [608, 30, 40, 120]], np.int64)
    fake = C.c_void_p(1 << 20)
    raw = _tables(lib, [(10, 20), (30, 40)], 32, 32, True, [2, 4])
    it = np.array([4, 2], np.int32)                  # same table size, other interpolations
    rc = lib.lib.yb_resize_batch_interp(fake, 1 << 20, desc.ctypes.data_as(C.c_void_p), fake, 2, 32, 32, 1,
                                        it.ctypes.data_as(C.c_void_p), raw.ctypes.data_as(C.c_void_p), fake, len(raw),
                                        fake, None, None)
    assert rc == -1 and b"another" in lib.lib.yb_last_error_string()


def test_python_entry_rejects_bad_interp_before_device_work():
    from yolov3_tensorflow_b200.utils import data_aug as A
    packed = A.PackedImages.__new__(A.PackedImages)
    packed.n, packed.device, packed.desc = 2, None, np.zeros((2, 4), np.int64)
    with pytest.raises(ValueError, match="image 1"):
        A._resize_packed_interp(packed, 32, 32, True, [2, 7])
    with pytest.raises(ValueError, match="3 interpolations"):
        A._resize_packed_interp(packed, 32, 32, True, [2, 3, 4])
