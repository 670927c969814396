"""Drop-in overlay for src/lib/utils/post_process.py: ctdet / multi_pose back-projection and the ddd tail
(ddd_post_process: 2D back-projection, alpha, 3D location and rot_y) on the device (accepts the CUDA tensor returned
by the decode, or the reference's numpy array).  The ddd helpers ddd_post_process_2d / _3d, get_alpha and
get_pred_depth are the reference's host code and stay with it: keep the original file as post_process_ref.py next
to this one."""
from centernet_b200.post_process import ctdet_post_process, ddd_post_process, multi_pose_post_process  # noqa: F401
try:  # the per-step ddd helpers are not on the detector's path: served by the untouched reference code
    from .post_process_ref import ddd_post_process_2d, ddd_post_process_3d, get_alpha, get_pred_depth  # noqa: F401
except ImportError:  # pragma: no cover
    pass
