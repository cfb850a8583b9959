"""CPU tests of the drawing path: the numpy restatement (tests/plot_ref.py) against the reference's goldens and, when
cv2 is importable, live OpenCV; the C-ABI label layout and score formatting against Python."""
import hashlib
import os

import numpy as np
import pytest

from tests import plot_cases, plot_ref as R

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plot.npz"))


def _draw_ref(seed):
    img, calls = plot_cases.case(seed)
    for coord, label, color, lt in calls:
        R.plot_one_box(img, coord, label=label, color=color, line_thickness=lt)
    return img


def test_restatement_equals_goldens():
    for s, h in zip(GOLDEN["seeds"].tolist(), GOLDEN["sha256"].tolist()):
        img = _draw_ref(s)
        assert hashlib.sha256(img.tobytes()).hexdigest() == h, f"seed {s}"
        if f"full_{s}" in GOLDEN.files:
            assert np.array_equal(img, GOLDEN[f"full_{s}"])


def test_restatement_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    for s in range(1000, 3000):
        img, calls = plot_cases.case(s)
        ref = img.copy()
        for coord, label, color, lt in calls:
            R.plot_one_box(img, coord, label=label, color=color, line_thickness=lt)
            # the reference's plot_one_box, spelled out with cv2 so no reference source is needed
            tl = lt or int(round(0.002 * max(ref.shape[0:2])))
            c1, c2 = (int(coord[0]), int(coord[1])), (int(coord[2]), int(coord[3]))
            cv2.rectangle(ref, c1, c2, color, thickness=tl)
            if label:
                tf = max(tl - 1, 1)
                t_size = cv2.getTextSize(label, 0, fontScale=float(tl) / 3, thickness=tf)[0]
                cv2.rectangle(ref, c1, (c1[0] + t_size[0], c1[1] - t_size[1] - 3), color, -1)
                cv2.putText(ref, label, (c1[0], c1[1] - 2), 0, float(tl) / 3, [0, 0, 0], thickness=tf,
                            lineType=cv2.LINE_AA)
        assert np.array_equal(img, ref), f"seed {s}"
    # order matters: the same boxes drawn the other way round give other pixels
    img, calls = plot_cases.case(1003)
    a, b = img.copy(), img.copy()
    for coord, label, color, lt in calls + [(calls[0][0] + 3, "person, 50.00%", [0, 0, 255], None)]:
        R.plot_one_box(a, coord, label=label, color=color, line_thickness=lt)
    for coord, label, color, lt in [(calls[0][0] + 3, "person, 50.00%", [0, 0, 255], None)] + calls:
        R.plot_one_box(b, coord, label=label, color=color, line_thickness=lt)
    assert not np.array_equal(a, b)


def test_text_codes_match_cv2_bytes():
    cv2 = pytest.importorskip("cv2")
    for s in plot_cases.NAMES + ["é?", "??", "\x7f", "\x01a"]:
        assert cv2.getTextSize(s, 0, 1.0, 1)[0] == R.text_size(R.text_codes(s), 1.0, 1), repr(s)
    assert cv2.getTextSize("é?", 0, 1.0, 1)[0][0] == 55


def test_layout_abi_equals_restatement():
    from yolov3_tensorflow_b200.utils.plot_utils import label_layout
    cv2 = None
    try:
        import cv2
    except ImportError:
        pass
    rng = np.random.default_rng(11)
    for k in range(3000):
        name = plot_cases.NAMES[k % len(plot_cases.NAMES)]
        tl = int(rng.integers(0, 3)) if k % 5 else int(rng.integers(3, 40))
        c1 = (int(rng.integers(-5000, 5000)), int(rng.integers(-5000, 5000)))
        score = np.float32(rng.random()) if k % 2 else None
        got = label_layout(name, tl, c1, score)
        label = name + (R.score_text(score) if score is not None else "")
        codes = R.text_codes(label)
        t_size, c2, org, tf = R.label_layout(codes, tl, c1)
        assert got["text"] == "".join(map(chr, codes))
        assert (got["t_size"], got["c2"], got["org"], got["thickness"]) == (t_size, c2, org, tf), (label, tl)
        if cv2 is not None:
            assert cv2.getTextSize(label, 0, float(tl) / 3, tf)[0] == t_size


def _abi_score(s):
    from yolov3_tensorflow_b200.utils.plot_utils import label_layout
    return label_layout("", 1, (0, 0), s)["text"]


def test_score_format_equals_python():
    rng = np.random.default_rng(3)
    vals = rng.random(1_000_000, dtype=np.float32)
    for v in vals:
        assert _abi_score(v) == ", {:.2f}%".format(v * np.float32(100)), v


def test_score_format_ties_and_specials():
    # every float32 in [0, 1] whose product with 100 is a decimal tie x.xx5 exactly: the product must be a multiple
    # of 1/200 with an odd numerator; products are float32 values, so walk the products and check their sources
    ties = []
    for num in range(1, 20000, 2):
        p = np.float32(num / 200)
        if float(p) == num / 200:
            # the float32 neighbours of p / 100 that map onto p
            s = np.float32(p / np.float32(100))
            for q in (np.nextafter(s, np.float32(0)), s, np.nextafter(s, np.float32(2))):
                if q * np.float32(100) == p and 0 <= q <= 1:
                    ties.append(q)
    assert len(ties) > 100
    special = [0.0, -0.0, 1.0, 1e-45, 1e-38, -1e-45, -1e-7, -0.004999, -0.00005, 0.99995, 0.999949, 0.5, 1e30,
               -3.4e38, 3.4e38, float("inf"), float("-inf"), float("nan"), 2.0 ** -30, 123456.789]
    for v in ties + [np.float32(x) for x in special]:
        assert _abi_score(v) == ", {:.2f}%".format(np.float32(v) * np.float32(100)), repr(v)


def test_pack_rejects_bad_sizes():
    import ctypes as C
    from yolov3_tensorflow_b200 import _lib
    nb = C.c_size_t()
    assert _lib.lib.yb_plot_workspace_bytes(1, 1, 3, C.byref(nb)) == 0
    buf = (C.c_uint8 * nb.value)()
    tl = (C.c_int * 1)(3)
    col = (C.c_int * 3)(1, 2, 3)
    ln = (C.c_int * 1)(3)
    assert _lib.lib.yb_plot_pack(tl, 1, col, b"dog", ln, 1, 1, buf, nb.value) == 0
    tl[0] = 1024
    assert _lib.lib.yb_plot_pack(tl, 1, col, b"dog", ln, 1, 1, buf, nb.value) == -1
    assert b"thickness" in _lib.lib.yb_last_error_string()
    tl[0] = 3
    ln[0] = 256
    assert _lib.lib.yb_plot_pack(tl, 1, col, b"dog", ln, 1, 1, buf, nb.value) == -1
    assert _lib.lib.yb_plot_pack(tl, 1, col, b"dog", ln, 1, 1, buf, 8) == -1
