"""mv_lm_icp_b200 -- H100-native multiview LM-ICP engine (hot path of adrelino/mv-lm-icp).

The product is the C-ABI library libmvicp.so (include/mvicp.h, csrc/); this package is its Python host mirror:
`Engine` wraps a context, `Frame` / `ICP_Ceres`-style helpers follow the reference's names (include/frame.h,
include/icp-ceres.h) so that the parity tests read like the reference's drivers."""
from ._lib import LmOptions, LmSummary, MvicpError, Stats, build, lib  # noqa: F401
from .api import (COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, TERMINATION, Engine, Frame,  # noqa: F401
                  ICP_Ceres, nccl_unique_id)
