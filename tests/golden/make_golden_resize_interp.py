"""Golden vectors for the training resize (yb_resize_batch_interp, resize_train_batch, resize_with_bbox with interp
2..4), produced by the REFERENCE's own utils/data_aug.resize_with_bbox (and so letterbox_resize) under OpenCV 4.13 on
the seeded cases of tests/resize_interp_cases.py, letterboxed and stretched, with INTER_CUBIC, INTER_AREA and
INTER_LANCZOS4.  INTER_CUBIC runs twice: as cv2 runs it by default (Intel IPP on, key prefix ipp_) and after
cv2.ipp.setUseIPP(False) (OpenCV's own code, the exact target).  Small results are stored in full with their boxes,
every result as a SHA-256; the cv2, numpy and IPP versions are recorded.
Run in the build container only:  YOLOV3_TF_REFERENCE=<checkout> python tests/golden/make_golden_resize_interp.py"""
import hashlib
import os
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import resize_interp_cases as K  # noqa: E402

sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))       # utils/*.py import it at module level
REF = os.environ["YOLOV3_TF_REFERENCE"]
sys.path.insert(0, REF)
from utils import data_aug  # noqa: E402


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    out = {"cv2_version": np.asarray(cv2.__version__), "numpy_version": np.asarray(np.__version__),
           "ipp_version": np.asarray(str(cv2.ipp.getIppVersion()))}
    cases = K.cases()
    out["cases"] = np.asarray([c for _, c, _ in cases], np.int64)
    keys, hashes, src_hashes = [], [], []
    for i, (sh, sw, nw, nh), full in cases:
        img = K.source(i, (sh, sw))
        src_hashes.append(_sha(img))
        gt = K.boxes(i, sh, sw)
        for interp in K.INTERPS:
            for lb in (True, False):
                runs = [("", False)] + ([("ipp_", True)] if interp == 2 else [])
                for prefix, ipp in runs:
                    cv2.ipp.setUseIPP(ipp if interp == 2 else True)
                    im, b = data_aug.resize_with_bbox(img, gt.copy(), nw, nh, interp=interp, letterbox=lb)  # REFERENCE
                    key = f"{prefix}{'lb' if lb else 'st'}{interp}_{i}"
                    keys.append(key)
                    hashes.append(_sha(im))
                    if full:
                        out[key] = im
                        if not prefix:
                            out[f"box_{key}"] = b
    cv2.ipp.setUseIPP(True)
    out["keys"], out["sha256"], out["src_sha256"] = np.asarray(keys), np.asarray(hashes), np.asarray(src_hashes)
    np.savez_compressed(os.path.join(HERE, "resize_interp.npz"), **out)


if __name__ == "__main__":
    main()
