"""GPU tests of the device drawing (yb_plot_boxes): every golden case, a mixed batch against single calls and the
restatement, decode -> draw -> encode without leaving the device, no synchronisation with check=False, and the
status of invalid detections."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import plot_cases, plot_ref as R

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "plot.npz"))


def _first_difference(seed, got):
    """How the device image differs from the restatement: the number of pixels and the first one."""
    img, calls = plot_cases.case(seed)
    for coord, label, color, lt in calls:
        R.plot_one_box(img, coord, label=label, color=color, line_thickness=lt)
    d = np.argwhere((img != got).any(2))
    return f"seed {seed}: {len(d)} pixels differ from the restatement, first at {d[:1].tolist()}"


def test_goldens_byte_identical():
    from yolov3_tensorflow_b200.utils.plot_utils import plot_one_box
    for s, h in zip(GOLDEN["seeds"].tolist(), GOLDEN["sha256"].tolist()):
        img, calls = plot_cases.case(s)
        t = torch.from_numpy(img).cuda()
        for coord, label, color, lt in calls:
            plot_one_box(t, coord, label=label, color=color, line_thickness=lt)
        got = t.cpu().numpy()
        assert hashlib.sha256(got.tobytes()).hexdigest() == h, _first_difference(s, got)
    img, calls = plot_cases.case(17)                     # the numpy path: one upload, one download per call
    for coord, label, color, lt in calls:
        plot_one_box(img, coord, label=label, color=color, line_thickness=lt)
    assert np.array_equal(img, GOLDEN["full_17"])


def _batch(n, seed, max_dets):
    r = np.random.default_rng(seed)
    imgs, boxes, scores, labels, counts = [], [], [], [], []
    slots = max_dets
    for i in range(n):
        h, w = int(r.integers(16, 900)), int(r.integers(16, 1200))
        imgs.append(r.integers(0, 256, (h, w, 3), dtype=np.uint8))
        c = int(r.integers(0, max_dets + 1))
        x = r.uniform(-0.3 * w, 1.3 * w, (slots, 2))
        y = r.uniform(-0.3 * h, 1.3 * h, (slots, 2))
        boxes.append(np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1).astype(np.float32))
        scores.append(r.random(slots, dtype=np.float32))
        labels.append(r.integers(0, 80, slots).astype(np.int32))
        counts.append(c)
    return imgs, np.stack(boxes), np.stack(scores), np.stack(labels), np.array(counts, np.int32)


def test_mixed_batch_equals_single_calls_and_restatement():
    from yolov3_tensorflow_b200.utils.plot_utils import get_color_table, plot_detections, plot_one_box
    imgs, boxes, scores, labels, counts = _batch(64, 1, 200)
    names = plot_cases.COCO
    table = get_color_table(80)
    packed = plot_detections(imgs, torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(),
                             torch.from_numpy(labels).cuda(), torch.from_numpy(counts).cuda(), names, table)
    for i, im in enumerate(imgs):
        got = packed.image(i).cpu().numpy()
        single = torch.from_numpy(im).cuda()
        for j in range(counts[i]):
            plot_one_box(single, boxes[i, j], label=names[labels[i, j]] + R.score_text(scores[i, j]),
                         color=table[labels[i, j]])
        assert np.array_equal(got, single.cpu().numpy()), f"image {i}"
        if i < 6:                                        # the restatement is slow: a few images, all detections
            ref = R.draw_detections(im.copy(), boxes[i, :counts[i]], scores[i, :counts[i]], labels[i, :counts[i]],
                                    names, table)
            assert np.array_equal(got, ref), f"image {i} vs restatement"


def test_decode_detect_draw_encode_on_device():
    """decode_jpeg_batch -> preprocess_batch -> detect_raw -> restore_boxes -> plot_detections -> encode_jpeg_batch,
    each image at the reference's own thickness (dog.jpg tl 1, messi.jpg tl 3), against the host copy of the same
    detections drawn by the restatement and encoded from the host."""
    from oracle import yolov3_oracle as O
    import yolov3_tensorflow_b200 as pkg
    from yolov3_tensorflow_b200.utils.data_aug import decode_jpeg_batch, encode_jpeg_batch, preprocess_batch, \
        restore_boxes
    from yolov3_tensorflow_b200.utils.plot_utils import get_color_table, plot_detections
    files = [os.path.join(HERE, "golden", f) for f in ("dog.jpg", "messi.jpg")]
    packed = decode_jpeg_batch(files)
    host = [packed.image(i).cpu().numpy() for i in range(2)]
    m = pkg.yolov3(80, O.COCO_ANCHORS, dtype="fp16")
    m.set_params(O.make_params(80, seed=7, random_bn=True, det_scale=8.0, conf_bias=-2.0), "HWIO")
    x, params = preprocess_batch(packed, 416, 416)
    _, out_boxes, out_scores, out_labels, _, counts = m.detect_raw(x, max_boxes=200, score_thresh=0.3, nms_thresh=0.45)
    counts = counts.clamp(max=12)                         # the restatement of thick text is slow on the host
    boxes = restore_boxes(out_boxes, counts, params)
    table = get_color_table(80)
    plot_detections(packed, boxes, out_scores, out_labels, counts, plot_cases.COCO, table)
    files_dev = encode_jpeg_batch(packed, quality=95)
    k = counts.cpu().tolist()
    assert min(k) > 0, f"no detections to draw: {k}"
    b, s, lab = boxes.cpu().numpy(), out_scores.cpu().numpy(), out_labels.cpu().numpy()
    for i, im in enumerate(host):
        ref = R.draw_detections(im.copy(), b[i, :k[i]], s[i, :k[i]], lab[i, :k[i]], plot_cases.COCO, table)
        got = packed.image(i).cpu().numpy()
        assert np.array_equal(got, ref), f"image {i}: {int((got != ref).any(2).sum())} pixels differ"
        assert files_dev[i] == encode_jpeg_batch([ref], quality=95)[0]


def test_check_false_does_not_sync():
    from yolov3_tensorflow_b200.utils.plot_utils import plot_detections
    imgs, boxes, scores, labels, counts = _batch(8, 2, 20)
    args = [torch.from_numpy(a).cuda() for a in (boxes, scores, labels, counts)]
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)                       # keep the stream busy: a sync would wait for it
    ev = torch.cuda.Event()
    ev.record()
    packed = plot_detections(imgs, *args, plot_cases.COCO, check=False)
    assert not ev.query(), "plot_detections(check=False) waited for the stream"
    torch.cuda.synchronize()
    assert (packed.plot_status[:, 0] == 0).all()


def test_invalid_detections_set_status():
    from yolov3_tensorflow_b200.utils.plot_utils import get_color_table, plot_detections
    imgs, boxes, scores, labels, counts = _batch(3, 3, 10)
    counts[:] = 10
    labels[0, 4] = 80
    labels[0, 6] = -1
    boxes[1, 2, 3] = np.nan
    boxes[1, 7, 0] = np.inf
    table = get_color_table(80)
    args = [torch.from_numpy(a).cuda() for a in (boxes, scores, labels, counts)]
    packed = plot_detections([im.copy() for im in imgs], *args, plot_cases.COCO, table, check=False)
    st = packed.plot_status.cpu().numpy()
    assert st.tolist() == [[1, 4], [2, 2], [0, -1]]
    for i in range(3):                                   # the rest is drawn as the reference would
        keep = [j for j in range(10) if 0 <= labels[i, j] < 80 and np.isfinite(boxes[i, j]).all()]
        ref = R.draw_detections(imgs[i].copy(), boxes[i, keep], scores[i, keep], labels[i, keep], plot_cases.COCO,
                                table)
        assert np.array_equal(packed.image(i).cpu().numpy(), ref)
    with pytest.raises(ValueError, match="image 0: detection 4"):
        plot_detections([im.copy() for im in imgs], *args, plot_cases.COCO, table)
