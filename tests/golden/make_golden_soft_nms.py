"""Generates tests/golden/soft_nms_ref.npz: the UNMODIFIED reference soft_nms (src/lib/external/nms.pyx, compiled by
oracle/build_ref.py into oracle/_ref/) on the seeded box lists of tests/test_post.py::test_reference_nms_module.
Build container only; the test reads the .npz.

    python tests/golden/make_golden_soft_nms.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref  # noqa: E402
from test_post import SOFT_NMS_LIVE, soft_nms_live_boxes  # noqa: E402

ref = build_ref.load_nms()
if ref is None:
    raise SystemExit("oracle/_ref nms module not built (python -m oracle.build_ref, where the reference exists)")
out = {}
for i, (method, Nt) in enumerate(SOFT_NMS_LIVE):
    b = soft_nms_live_boxes(i)
    a = b.copy()
    keep = ref.soft_nms(a, Nt=Nt, method=method)
    out["boxes_out_%d" % i] = a
    out["keep_%d" % i] = np.asarray(keep, dtype=np.int64)
np.savez_compressed(os.path.join(HERE, "soft_nms_ref.npz"), **out)
print("wrote", len(out), "arrays")
