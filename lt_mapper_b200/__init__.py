"""H100-native LT-removert / LT-map hot path (see DESIGN.md).

`binding` is the ctypes view of the C-ABI (include/ltr_b200.h); `removert` mirrors the reference's
Removerter / Session call graph on top of it.  CUDA-only: importing works anywhere, but creating a
context without libltr_b200.so or without an sm_90 GPU raises.
"""
from . import binding  # noqa: F401
from .binding import Context, LtrError, MODE_HD, MODE_ND, MODE_PD, SCANSIDE_MAP, SCANSIDE_SCAN_MINUS_MAP, reset_rimg_size  # noqa: F401
from .binding import ICP_ITERATIONS, ICP_TRANSFORM, ICP_ABS_MSE, ICP_REL_MSE, ICP_NO_CORRESPONDENCES  # noqa: F401
