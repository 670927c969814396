"""centernet_b200 -- H100-native (sm_90a) CenterNet heat-map hot path.

Host-side mirror of the reference operator interface:

  centernet_b200.decode    <->  src/lib/models/decode.py
  centernet_b200.utils     <->  src/lib/models/utils.py
  centernet_b200.losses    <->  src/lib/models/losses.py
  centernet_b200.dcn_v2 / dcn_v2_func  <->  src/lib/models/networks/DCNv2/

Every op runs hand-written CUDA through the C ABI of ``include/centernet_b200.h``;
there is no CPU or eager-PyTorch fallback: importing without the built extension, or
calling with non-CUDA tensors, raises.
"""
from ._lib import C as _C, version  # noqa: F401  (fails loudly if the extension is missing)

__all__ = ["decode", "utils", "losses", "dcn_v2", "dcn_v2_func", "heads", "ida", "version"]
