"""mv_lm_icp_b200 -- H100-native multiview LM-ICP engine (hot path of adrelino/mv-lm-icp).

The product is the C-ABI library libmvicp.so (include/mvicp.h, csrc/); this package is its Python host mirror:
`Engine` wraps a context, `Frame` / `ICP_Ceres`-style helpers follow the reference's names (include/frame.h,
include/icp-ceres.h) so that the parity tests read like the reference's drivers."""
from ._lib import G2oOptions, G2oSummary, LmOptions, LmSummary, MvicpError, Stats, build, lib  # noqa: F401
from .api import (COV_FIXED, COV_INDEPENDENT, COV_OK, COV_SINGULAR, COST_MIXED, COST_P2P, COST_P2PLANE, PARAM_AA, PARAM_QUAT, PARAM_SE3, TERMINATION, DeviceEdges, Engine,  # noqa: F401
                  Frame, ICP_Ceres, ICP_G2O, default_g2o_options, nccl_unique_id)
