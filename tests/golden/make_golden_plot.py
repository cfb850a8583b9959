"""Golden data for the drawing tests: the reference's own utils/plot_utils.py drawn with OpenCV over the seeded
cases of tests/plot_cases.py.  Stores the SHA-256 of every result image, a few small results in full, and the
OpenCV and NumPy versions, in plot.npz.

    python tests/golden/make_golden_plot.py /path/to/reference
"""
import hashlib
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import plot_cases  # noqa: E402

SEEDS = range(400)
FULL = (17, 34)


def main(ref):
    sys.path.insert(0, os.path.join(ref, "utils"))
    import plot_utils
    out = {"cv2_version": np.array(cv2.__version__), "numpy_version": np.array(np.__version__),
           "seeds": np.array(list(SEEDS), np.int32)}
    hashes = []
    for s in SEEDS:
        img, calls = plot_cases.case(s)
        for coord, label, color, lt in calls:
            plot_utils.plot_one_box(img, coord, label=label, color=color, line_thickness=lt)
        hashes.append(hashlib.sha256(img.tobytes()).hexdigest())
        if s in FULL:
            out[f"full_{s}"] = img
    out["sha256"] = np.array(hashes)
    np.savez_compressed(os.path.join(HERE, "plot.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1])
