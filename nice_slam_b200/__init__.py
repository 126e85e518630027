"""nice_slam_b200 -- H100 (sm_90a) render-and-backprop path for NICE-SLAM (drop-in for src/utils/Renderer.py).

Public surface:
    FusedRenderer   mirror of the reference's Renderer (render_batch_ray / eval_points / render_img)
    NICEDecoders    parameter container with the reference's state_dict keys
    FusedMapper     one Mapper.optimize_map call on the fused path (mapping.py)
    FusedSLAM       a whole RGB-D sequence on the fused path, NICE_SLAM.run under strict sync (slam.py); ate_rmse
    to_channels_last, lib (ctypes handle of libnsb.so)
"""
from ._lib import lib, LIB_PATH                       # noqa: F401
from .decoders import NICEDecoders                     # noqa: F401
from .renderer import FusedRenderer, to_channels_last  # noqa: F401
from .mapping import FusedMapper                       # noqa: F401
from .slam import FusedSLAM, ate_rmse                  # noqa: F401

__all__ = ["FusedRenderer", "FusedMapper", "FusedSLAM", "ate_rmse", "NICEDecoders", "to_channels_last", "lib", "LIB_PATH"]
