"""Drop-in overlay for src/lib/models/decode.py of xingyizhou/CenterNet.

Copy (or symlink) this file over the reference's src/lib/models/decode.py with
`centernet_b200` importable (e.g. `pip install -e <repo>` or PYTHONPATH=<repo>).  Every name the
reference module exports is re-exported with the same signature, so detectors/*.py and trains/*.py
keep working unchanged (they do `from models.decode import ctdet_decode`, ...)."""
from centernet_b200.decode import (  # noqa: F401
    _nms, _topk, _topk_channel, _left_aggregate, _right_aggregate, _top_aggregate, _bottom_aggregate,
    _h_aggregate, _v_aggregate, agnex_ct_decode, exct_decode, ddd_decode, ctdet_decode, multi_pose_decode,
    _gather_feat, _transpose_and_gather_feat,
    # extras: fused-sigmoid variants (INTEGRATION.md section 1)
    ctdet_decode_from_logits, multi_pose_decode_from_logits, ddd_decode_from_logits, exct_decode_from_logits,
    agnex_ct_decode_from_logits)
